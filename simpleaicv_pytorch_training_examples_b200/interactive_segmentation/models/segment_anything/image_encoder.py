"""SAM ViT image encoder with the reference's constructor surface and state_dict layout
(SimpleAICV/interactive_segmentation/models/segment_anything/image_encoder.py:8-29 PatchEmbed, :147-184 Attention,
:187-198 MLPBlock, :201-239 Block, :242-256 LayerNorm2d, :259-331 ViTImageEncoder), executed by
engine.sam.SamEncoderRT on sm_90a kernels (wgmma GEMMs and attention with the decomposed rel-pos bias in the
score GEMM).  The nn.Modules are parameter containers created in the reference's order."""
import torch
import torch.nn as nn

from ....engine.convnet import run_network
from ....engine.sam import SamEncoderRT


class PatchEmbed(nn.Module):

    def __init__(self, inplanes=3, planes=768, kernel_size=16, stride=16, padding=0):
        super().__init__()
        assert padding == 0 and kernel_size == stride
        self.proj = nn.Conv2d(inplanes, planes, kernel_size=kernel_size, stride=stride, padding=padding)


class Attention(nn.Module):

    def __init__(self, inplanes, head_nums=8, input_size=None):
        super().__init__()
        self.head_nums = head_nums
        head_planes = inplanes // head_nums
        self.scale = head_planes ** -0.5
        self.qkv = nn.Linear(inplanes, inplanes * 3)
        self.proj = nn.Linear(inplanes, inplanes)
        assert input_size is not None, 'Input size must be provided if using relative positional encoding.'
        self.rel_pos_h = nn.Parameter(torch.zeros(2 * input_size[0] - 1, head_planes))
        self.rel_pos_w = nn.Parameter(torch.zeros(2 * input_size[1] - 1, head_planes))


class MLPBlock(nn.Module):

    def __init__(self, inplanes, mlp_planes):
        super().__init__()
        self.lin1 = nn.Linear(inplanes, mlp_planes)
        self.lin2 = nn.Linear(mlp_planes, inplanes)
        self.act = nn.GELU()


class Block(nn.Module):

    def __init__(self, inplanes, head_nums, mlp_ratio=4.0, input_size=None, window_size=0):
        super().__init__()
        self.norm1 = nn.LayerNorm(inplanes, eps=1e-6)
        self.attn = Attention(inplanes=inplanes, head_nums=head_nums,
                              input_size=input_size if window_size == 0 else (window_size, window_size))
        self.norm2 = nn.LayerNorm(inplanes, eps=1e-6)
        self.mlp = MLPBlock(inplanes=inplanes, mlp_planes=int(inplanes * mlp_ratio))
        self.window_size = window_size


class LayerNorm2d(nn.Module):

    def __init__(self, inplanes, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(inplanes))
        self.bias = nn.Parameter(torch.zeros(inplanes))
        self.eps = eps


class ViTImageEncoder(nn.Module):

    def __init__(self, image_size=1024, patch_size=16, inplanes=3, embedding_planes=768, block_nums=12, head_nums=12, mlp_ratio=4,
                 out_planes=256, window_size=0, global_attn_indexes=(), use_gradient_checkpoint=False):
        super().__init__()
        self.image_size = image_size
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.patch_embed = PatchEmbed(inplanes=inplanes, planes=embedding_planes, kernel_size=patch_size, stride=patch_size, padding=0)
        self.pos_embed = nn.Parameter(torch.zeros(1, image_size // patch_size, image_size // patch_size, embedding_planes))
        grid = image_size // patch_size
        self.blocks = nn.ModuleList([
            Block(inplanes=embedding_planes, head_nums=head_nums, mlp_ratio=mlp_ratio, input_size=(grid, grid),
                  window_size=window_size if i not in global_attn_indexes else 0) for i in range(block_nums)])
        self.neck = nn.Sequential(nn.Conv2d(embedding_planes, out_planes, kernel_size=1, stride=1, padding=0, bias=False),
                                  LayerNorm2d(out_planes),
                                  nn.Conv2d(out_planes, out_planes, kernel_size=3, stride=1, padding=1, bias=False),
                                  LayerNorm2d(out_planes))

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            rt = SamEncoderRT(self)
            self.__dict__['_rt'] = rt
        return rt

    def grad_sink(self):
        return self._runtime().sink

    def forward(self, x):
        """x: fp32 [B, 3, S, S] -> fp32 [B, out_planes, S/patch, S/patch]"""
        if not x.is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU (no CPU fallback exists)')
        return run_network(self._runtime(), x.float(), self.training)
