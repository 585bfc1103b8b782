"""ViT-B/L/H with the reference's constructor surface and state_dict layout
(SimpleAICV/classification/backbones/vit.py:18-47 PatchEmbeddingBlock, :50-80 MultiHeadAttention,
:83-99 FeedForward, :138-163 TransformerEncoderLayer, :166-262 ViT, :273-282 constructors),
executed by engine.vit.ViTRT on hand-written sm_90a kernels.

The nn.Modules are parameter containers built in the reference's order (identical seeded init and
state_dict keys); ``forward`` hands the batch to the runtime.  CPU tensors raise.
"""
import torch
import torch.nn as nn

from ...engine.runtime import RuntimeModule
from ...engine.vit import ViTRT

__all__ = ['vit_base_patch16', 'vit_large_patch16', 'vit_huge_patch14']


class PatchEmbeddingBlock(nn.Module):

    def __init__(self, inplanes, planes, kernel_size, stride, padding, groups=1, has_norm=False):
        super().__init__()
        assert not has_norm and groups == 1 and padding == 0 and kernel_size == stride
        self.proj = nn.Conv2d(inplanes, planes, kernel_size, stride=stride, padding=padding, groups=groups, bias=True)
        self.norm = nn.Identity()


class MultiHeadAttention(nn.Module):

    def __init__(self, inplanes, head_nums=8, dropout_prob=0.):
        super().__init__()
        self.head_nums = head_nums
        self.scale = (inplanes // head_nums) ** -0.5
        self.qkv = nn.Linear(inplanes, inplanes * 3)
        self.proj = nn.Linear(inplanes, inplanes)
        self.dropout = nn.Dropout(dropout_prob)
        self.softmax = nn.Softmax(dim=-1)


class FeedForward(nn.Module):

    def __init__(self, inplanes, feedforward_planes, dropout_prob=0.):
        super().__init__()
        self.fc1 = nn.Linear(inplanes, feedforward_planes)
        self.gelu = nn.GELU()
        self.fc2 = nn.Linear(feedforward_planes, inplanes)
        self.drop = nn.Dropout(dropout_prob)


class DropPathBlock(nn.Module):
    """Stochastic depth marker (vit.py:102-135); the per-sample mask is drawn by the runtime."""

    def __init__(self, drop_path_prob=0., scale_by_keep=True):
        super().__init__()
        assert drop_path_prob >= 0.
        self.drop_path_prob = drop_path_prob
        self.keep_path_prob = 1 - drop_path_prob
        self.scale_by_keep = scale_by_keep


class TransformerEncoderLayer(nn.Module):

    def __init__(self, inplanes, head_nums, feedforward_ratio=4, dropout_prob=0., drop_path_prob=0.):
        super().__init__()
        self.norm1 = nn.LayerNorm(inplanes, eps=1e-6)
        self.attn = MultiHeadAttention(inplanes, head_nums, dropout_prob=dropout_prob)
        self.norm2 = nn.LayerNorm(inplanes, eps=1e-6)
        self.mlp = FeedForward(inplanes, int(inplanes * feedforward_ratio), dropout_prob=dropout_prob)
        self.drop_path = DropPathBlock(drop_path_prob) if drop_path_prob > 0. else nn.Identity()


class ViT(RuntimeModule):

    def __init__(self, patch_size, embedding_planes, block_nums, head_nums, feedforward_ratio, image_size=224,
                 dropout_prob=0., drop_path_prob=0., global_pool=False, num_classes=1000,
                 use_gradient_checkpoint=False):
        super().__init__()
        self.image_size = image_size
        self.patch_size = patch_size
        self.embedding_planes = embedding_planes
        self.block_nums = block_nums
        self.head_nums = head_nums
        self.feedforward_ratio = feedforward_ratio
        self.global_pool = global_pool
        self.num_classes = num_classes
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.dropout_prob = dropout_prob
        self.patch_embed = PatchEmbeddingBlock(3, embedding_planes, kernel_size=patch_size, stride=patch_size, padding=0)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embedding_planes))
        self.pos_embed = nn.Parameter(torch.ones(1, (image_size // patch_size) ** 2 + 1, embedding_planes))
        self.embedding_dropout = nn.Dropout(dropout_prob)
        rates = [0. if drop_path_prob == 0. else drop_path_prob * (i / (block_nums - 1)) for i in range(block_nums)]
        self.blocks = nn.ModuleList([
            TransformerEncoderLayer(embedding_planes, head_nums, feedforward_ratio=feedforward_ratio,
                                    dropout_prob=dropout_prob, drop_path_prob=r) for r in rates])
        self.norm = nn.LayerNorm(embedding_planes, eps=1e-6)
        self.fc = nn.Linear(embedding_planes, num_classes)
        # vit.py:228-237
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        nn.init.normal_(self.cls_token, std=1e-6)
        nn.init.trunc_normal_(self.fc.weight, std=2e-5)
        nn.init.zeros_(self.fc.bias)

    def _build_runtime(self):
        return ViTRT(self)

    def forward(self, x):
        return self._run(x.float())


def _vit(patch_size, embedding_planes, block_nums, head_nums, feedforward_ratio, **kwargs):
    return ViT(patch_size, embedding_planes, block_nums, head_nums, feedforward_ratio, **kwargs)


def vit_base_patch16(**kwargs):
    return _vit(16, 768, 12, 12, 4, **kwargs)


def vit_large_patch16(**kwargs):
    return _vit(16, 1024, 24, 16, 4, **kwargs)


def vit_huge_patch14(**kwargs):
    return _vit(14, 1280, 32, 16, 4, **kwargs)
