"""VAN b0..b6 with the reference's constructor surface and state_dict layout
(SimpleAICV/classification/backbones/van.py:20-35 DWConv, :38-56 Mlp, :59-93 LKA, :96-115 Attention,
:118-151 DropPathBlock, :154-186 Block, :189-208 OverlapPatchEmbed, :211-310 VAN, :322-368 constructors),
executed by engine.van.VANRT on sm_90a kernels.  The nn.Modules are parameter containers created in the
reference's order (identical seeded init and state_dict keys); ``forward`` hands the batch to the runtime.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from ...engine.convnet import run_network
from ...engine.van import VANRT

__all__ = ['van_b0', 'van_b1', 'van_b2', 'van_b3', 'van_b4', 'van_b5', 'van_b6']


class DWConv(nn.Module):

    def __init__(self, inplanes=768):
        super().__init__()
        self.dwconv = nn.Conv2d(inplanes, inplanes, kernel_size=3, stride=1, padding=1, bias=True, groups=inplanes)


class Mlp(nn.Module):

    def __init__(self, inplanes, hidden_planes, planes, dropout_prob=0.):
        super().__init__()
        self.fc1 = nn.Conv2d(inplanes, hidden_planes, 1)
        self.dwconv = DWConv(hidden_planes)
        self.act = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(hidden_planes, planes, 1)
        self.drop = nn.Dropout(dropout_prob)


class LKA(nn.Module):

    def __init__(self, inplanes):
        super().__init__()
        self.conv0 = nn.Conv2d(inplanes, inplanes, kernel_size=5, stride=1, padding=2, groups=inplanes, bias=True)
        self.conv_spatial = nn.Conv2d(inplanes, inplanes, kernel_size=7, stride=1, padding=9, groups=inplanes, dilation=3,
                                      bias=True)
        self.conv1 = nn.Conv2d(inplanes, inplanes, kernel_size=1, stride=1, padding=0, bias=True)


class Attention(nn.Module):

    def __init__(self, inplanes):
        super().__init__()
        self.proj_1 = nn.Conv2d(inplanes, inplanes, 1)
        self.activation = nn.ReLU(inplace=True)
        self.spatial_gating_unit = LKA(inplanes)
        self.proj_2 = nn.Conv2d(inplanes, inplanes, 1)


class DropPathBlock(nn.Module):

    def __init__(self, drop_path_prob=0., scale_by_keep=True):
        super().__init__()
        assert drop_path_prob >= 0.
        self.drop_path_prob = drop_path_prob
        self.keep_path_prob = 1 - drop_path_prob
        self.scale_by_keep = scale_by_keep


class Block(nn.Module):

    def __init__(self, inplanes, mlp_ratio=4., dropout_prob=0., drop_path_prob=0.):
        super().__init__()
        self.norm1 = nn.BatchNorm2d(inplanes)
        self.attn = Attention(inplanes)
        self.norm2 = nn.BatchNorm2d(inplanes)
        self.mlp = Mlp(inplanes=inplanes, hidden_planes=int(inplanes * mlp_ratio), planes=inplanes, dropout_prob=dropout_prob)
        self.layer_scale_1 = nn.Parameter(1e-5 * torch.ones((1, inplanes, 1, 1)), requires_grad=True)
        self.layer_scale_2 = nn.Parameter(1e-5 * torch.ones((1, inplanes, 1, 1)), requires_grad=True)
        self.drop_path = DropPathBlock(drop_path_prob) if drop_path_prob > 0. else nn.Identity()


class OverlapPatchEmbed(nn.Module):

    def __init__(self, patch_size=7, stride=4, inplanes=3, embedding_planes=768):
        super().__init__()
        self.proj = nn.Conv2d(inplanes, embedding_planes, kernel_size=patch_size, stride=stride,
                              padding=(patch_size // 2, patch_size // 2))
        self.norm = nn.BatchNorm2d(embedding_planes)


class VAN(nn.Module):

    def __init__(self, inplanes=3, embedding_planes=[64, 128, 256, 512], mlp_ratios=[4, 4, 4, 4], block_nums=[3, 4, 6, 3],
                 dropout_prob=0., drop_path_prob=0., num_classes=1000, use_gradient_checkpoint=False):
        super().__init__()
        assert len(embedding_planes) == len(mlp_ratios) == len(block_nums)
        self.block_nums = block_nums
        self.num_classes = num_classes
        self.use_gradient_checkpoint = use_gradient_checkpoint
        rates = [x for x in np.linspace(0, drop_path_prob, sum(block_nums))]
        idx, cur = 0, inplanes
        for i in range(len(block_nums)):
            pe = OverlapPatchEmbed(patch_size=7 if i == 0 else 3, stride=4 if i == 0 else 2, inplanes=cur,
                                   embedding_planes=embedding_planes[i])
            cur = embedding_planes[i]
            block = nn.ModuleList([Block(inplanes=embedding_planes[i], mlp_ratio=mlp_ratios[i], dropout_prob=dropout_prob,
                                         drop_path_prob=rates[idx + j]) for j in range(block_nums[i])])
            norm = nn.BatchNorm2d(embedding_planes[i])
            idx += block_nums[i]
            setattr(self, f'patch_embed{i + 1}', pe)
            setattr(self, f'block{i + 1}', block)
            setattr(self, f'norm{i + 1}', norm)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.head = nn.Linear(embedding_planes[3], num_classes)
        for m in self.modules():  # van.py:265-279
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.Conv2d):
                fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                fan_out //= m.groups
                m.weight.data.normal_(0, math.sqrt(2.0 / fan_out))
                if m.bias is not None:
                    m.bias.data.zero_()

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            rt = VANRT(self)
            self.__dict__['_rt'] = rt
        return rt

    def grad_sink(self):
        return self._runtime().sink

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU (no CPU fallback exists)')
        return run_network(self._runtime(), x.float(), self.training)


def _van(embedding_planes, mlp_ratios, block_nums, **kwargs):
    return VAN(embedding_planes=embedding_planes, mlp_ratios=mlp_ratios, block_nums=block_nums, **kwargs)


def van_b0(**kwargs):
    return _van([32, 64, 160, 256], [8, 8, 4, 4], [3, 3, 5, 2], **kwargs)


def van_b1(**kwargs):
    return _van([64, 128, 320, 512], [8, 8, 4, 4], [2, 2, 4, 2], **kwargs)


def van_b2(**kwargs):
    return _van([64, 128, 320, 512], [8, 8, 4, 4], [3, 3, 12, 3], **kwargs)


def van_b3(**kwargs):
    return _van([64, 128, 320, 512], [8, 8, 4, 4], [3, 5, 27, 3], **kwargs)


def van_b4(**kwargs):
    return _van([64, 128, 320, 512], [8, 8, 4, 4], [3, 6, 40, 3], **kwargs)


def van_b5(**kwargs):
    return _van([96, 192, 480, 768], [8, 8, 4, 4], [3, 3, 24, 3], **kwargs)


def van_b6(**kwargs):
    return _van([96, 192, 384, 768], [8, 8, 4, 4], [6, 6, 90, 6], **kwargs)
