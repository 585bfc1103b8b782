"""DINOv3 ViT backbones with the reference's constructor surface, state_dict layout and seeded init
(SimpleAICV/detection/models/backbones/dinov3vit.py:35-71 PatchEmbed, :74-90 LayerScale, :93-141 Mlp / SwiGLUFFN,
:144-268 RopePositionEmbedding, :285-300 LinearKMaskedBias, :303-367 SelfAttention, :370-469 SelfAttentionBlock,
:472-572 DinoVisionTransformer, :575-715 constructors), executed by engine.dinov3.DINOv3RT on sm_90a kernels.  The
nn.Modules are parameter containers created in the reference's order, so ``torch.manual_seed`` gives the reference's
initial weights."""
import math

import torch
import torch.nn as nn

from ....classification.common import load_state_dict
from ....engine.dinov3 import DINOv3RT, rope_sincos
from ....engine.runtime import RuntimeModule

__all__ = [
    'dinov3_vit_small_patch16_backbone',
    'dinov3_vit_small_plus_patch16_backbone',
    'dinov3_vit_base_patch16_backbone',
    'dinov3_vit_large_patch16_backbone',
    'dinov3_vit_large_plus_patch16_backbone',
    'dinov3_vit_huge_plus_patch16_backbone',
    'dinov3_vit_7b_patch16_backbone',
]


class PatchEmbed(nn.Module):

    def __init__(self, inplanes=3, planes=768, kernel_size=16, stride=16, padding=0, has_norm=False):
        super().__init__()
        if has_norm or padding != 0 or kernel_size != stride:
            raise NotImplementedError('DINOv3 PatchEmbed: only the non-overlapping patch embedding without norm is built')
        self.planes = planes
        self.proj = nn.Conv2d(inplanes, planes, kernel_size=kernel_size, stride=stride, padding=padding)
        k = 1 / (inplanes * (kernel_size ** 2))
        nn.init.uniform_(self.proj.weight, -math.sqrt(k), math.sqrt(k))
        nn.init.uniform_(self.proj.bias, -math.sqrt(k), math.sqrt(k))


class LayerScale(nn.Module):

    def __init__(self, inplanes, init_values=1e-5):
        super().__init__()
        self.gamma = nn.Parameter(torch.empty(inplanes))
        nn.init.constant_(self.gamma, init_values)


class Mlp(nn.Module):

    def __init__(self, inplanes, hidden_planes, planes, bias=True):
        super().__init__()
        self.fc1 = nn.Linear(inplanes, hidden_planes, bias=bias)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_planes, planes, bias=bias)


class SwiGLUFFN(nn.Module):

    def __init__(self, inplanes, hidden_planes, planes, bias=True, align_to=8):
        super().__init__()
        d = int(hidden_planes * 2 / 3)
        swiglu_hidden_planes = d + (-d % align_to)
        self.w1 = nn.Linear(inplanes, swiglu_hidden_planes, bias=bias)
        self.w2 = nn.Linear(inplanes, swiglu_hidden_planes, bias=bias)
        self.w3 = nn.Linear(swiglu_hidden_planes, planes, bias=bias)


class RopePositionEmbedding(nn.Module):

    def __init__(self, embedding_planes, head_nums, base=100.0, min_period=None, max_period=None, normalize_coords='separate',
                 shift_coords=None, jitter_coords=None, rescale_coords=None):
        super().__init__()
        assert normalize_coords in ['min', 'max', 'separate']
        assert embedding_planes % (4 * head_nums) == 0
        both_periods = min_period is not None and max_period is not None
        if (base is None and not both_periods) or (base is not None and both_periods):
            raise ValueError('Either `base` or `min_period`+`max_period` must be provided.')
        if shift_coords is not None or jitter_coords is not None:
            raise NotImplementedError('DINOv3 RoPE shift_coords / jitter_coords are not implemented by the H100 runtime '
                                      '(None in every constructor)')
        head_planes = embedding_planes // head_nums
        self.min_period, self.max_period = min_period, max_period
        self.normalize_coords = normalize_coords
        self.shift_coords, self.jitter_coords, self.rescale_coords = shift_coords, jitter_coords, rescale_coords
        # persistent: checkpoints overwrite it, and the runtime reads it (never a closed form)
        self.register_buffer('periods', torch.empty(head_planes // 4), persistent=True)
        if base is not None:
            periods = base ** (2 * torch.arange(head_planes // 4) / (head_planes // 2))
        else:
            base = self.max_period / self.min_period
            periods = base ** torch.linspace(0, 1, head_planes // 4) / base * self.max_period
        self.periods.data = periods

    def forward(self, H, W):
        """(sin, cos) [H*W, head_planes], the reference's expression (one rescale draw per training call)."""
        return rope_sincos(self, H, W, self.training)


class LinearKMaskedBias(nn.Linear):

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        o = self.out_features
        assert o % 3 == 0
        if self.bias is not None:
            self.register_buffer('bias_mask', torch.full_like(self.bias, fill_value=1))
            self.bias_mask[o // 3:2 * o // 3].fill_(0)


class SelfAttention(nn.Module):

    def __init__(self, inplanes, head_nums=8, qkv_bias=False, proj_bias=True):
        super().__init__()
        self.head_nums = head_nums
        self.scale = (inplanes // head_nums) ** -0.5
        self.qkv = LinearKMaskedBias(inplanes, inplanes * 3, bias=qkv_bias)
        self.proj = nn.Linear(inplanes, inplanes, bias=proj_bias)


class SelfAttentionBlock(nn.Module):

    def __init__(self, inplanes, head_nums, ffn_ratio=4.0, qkv_bias=False, proj_bias=True, ffn_bias=True, init_values=None,
                 ffn_layer=Mlp):
        super().__init__()
        if not init_values:
            raise NotImplementedError('DINOv3 blocks without LayerScale (layerscale_init falsy) are not built (1e-5 in every '
                                      'constructor)')
        self.norm1 = nn.LayerNorm(inplanes, eps=1e-6)
        self.attn = SelfAttention(inplanes, head_nums=head_nums, qkv_bias=qkv_bias, proj_bias=proj_bias)
        self.ls1 = LayerScale(inplanes, init_values=init_values)
        self.norm2 = nn.LayerNorm(inplanes, eps=1e-6)
        self.mlp = ffn_layer(inplanes=inplanes, hidden_planes=int(inplanes * ffn_ratio), planes=inplanes, bias=ffn_bias)
        self.ls2 = LayerScale(inplanes, init_values=init_values)


class DinoVisionTransformer(RuntimeModule):

    def __init__(self, patch_size=16, inplanes=3, embedding_planes=768, pos_embed_rope_base=100.0, pos_embed_rope_min_period=None,
                 pos_embed_rope_max_period=None, pos_embed_rope_normalize_coords='separate', pos_embed_rope_shift_coords=None,
                 pos_embed_rope_jitter_coords=None, pos_embed_rope_rescale_coords=None, block_nums=12, head_nums=12, ffn_ratio=4.0,
                 qkv_bias=True, drop_path_rate=0., layerscale_init=1e-5, ffn_layer='mlp', ffn_bias=True, proj_bias=True,
                 use_gradient_checkpoint=False):
        super().__init__()
        assert pos_embed_rope_normalize_coords in ['min', 'max', 'separate']
        if drop_path_rate > 0.:
            raise NotImplementedError('DINOv3 drop_path_rate > 0 (the subset / index_add scheme of dinov3vit.py:436-464) is not '
                                      'implemented by the H100 runtime (0 in every shipped config)')
        if ffn_layer not in ('mlp', 'swiglu'):
            raise NotImplementedError(f'DINOv3 ffn_layer={ffn_layer!r} is not built (mlp and swiglu are)')
        self.patch_size = patch_size
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.patch_embed = PatchEmbed(inplanes=inplanes, planes=embedding_planes, kernel_size=patch_size, stride=patch_size,
                                      padding=0, has_norm=False)
        self.rope_embed = RopePositionEmbedding(embedding_planes=embedding_planes, head_nums=head_nums, base=pos_embed_rope_base,
                                                min_period=pos_embed_rope_min_period, max_period=pos_embed_rope_max_period,
                                                normalize_coords=pos_embed_rope_normalize_coords,
                                                shift_coords=pos_embed_rope_shift_coords, jitter_coords=pos_embed_rope_jitter_coords,
                                                rescale_coords=pos_embed_rope_rescale_coords)
        ffn_cls = {'mlp': Mlp, 'swiglu': SwiGLUFFN}[ffn_layer]
        self.blocks = nn.ModuleList([
            SelfAttentionBlock(inplanes=embedding_planes, head_nums=head_nums, ffn_ratio=ffn_ratio, qkv_bias=qkv_bias,
                               proj_bias=proj_bias, ffn_bias=ffn_bias, init_values=layerscale_init, ffn_layer=ffn_cls)
            for _ in range(block_nums)])
        self.norm = nn.LayerNorm(embedding_planes, eps=1e-6)
        self.out_channels = embedding_planes
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def _build_runtime(self):
        return DINOv3RT(self)

    def forward(self, x):
        """x: fp32 [B, 3, H, W] -> fp32 [B, C, H/patch, W/patch]"""
        return self._run(x.float())


def _dinov3vitbackbone(patch_size, embedding_planes, pos_embed_rope_normalize_coords, pos_embed_rope_rescale_coords, block_nums,
                       head_nums, ffn_ratio, qkv_bias, ffn_layer, pretrained_path='', **kwargs):
    model = DinoVisionTransformer(patch_size=patch_size, embedding_planes=embedding_planes,
                                  pos_embed_rope_normalize_coords=pos_embed_rope_normalize_coords,
                                  pos_embed_rope_rescale_coords=pos_embed_rope_rescale_coords, block_nums=block_nums,
                                  head_nums=head_nums, ffn_ratio=ffn_ratio, qkv_bias=qkv_bias, ffn_layer=ffn_layer, **kwargs)
    if pretrained_path:
        load_state_dict(pretrained_path, model)
    else:
        print('no backbone pretrained model!')
    return model


def dinov3_vit_small_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 384, 'separate', 2, 12, 6, 4, True, 'mlp', pretrained_path, **kwargs)


def dinov3_vit_small_plus_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 384, 'separate', 2, 12, 6, 6, True, 'swiglu', pretrained_path, **kwargs)


def dinov3_vit_base_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 768, 'separate', 2, 12, 12, 4, True, 'mlp', pretrained_path, **kwargs)


def dinov3_vit_large_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 1024, 'separate', 2, 24, 16, 4, True, 'mlp', pretrained_path, **kwargs)


def dinov3_vit_large_plus_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 1024, 'separate', 2, 24, 16, 6, True, 'swiglu', pretrained_path, **kwargs)


def dinov3_vit_huge_plus_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    return _dinov3vitbackbone(patch_size, 1280, 'separate', 2, 32, 20, 6, True, 'swiglu', pretrained_path, **kwargs)


def dinov3_vit_7b_patch16_backbone(patch_size=16, pretrained_path='', **kwargs):
    raise NotImplementedError('dinov3_vit_7b_patch16_backbone is not built: width 4096 and head size 128 are not supported by '
                              'the LayerNorm and attention kernels')
