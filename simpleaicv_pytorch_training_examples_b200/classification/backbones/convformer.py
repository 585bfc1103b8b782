"""ConvFormer S18 / S36 / M36 / B36 with the reference's constructor surface and state_dict layout
(SimpleAICV/classification/backbones/convformer.py:16-44 Downsampling, :47-79 SepConv, :82-103 Mlp, :106-139
DropPathBlock, :142-166 MetaFormerBlock, :169-256 MetaFormer, :259-296 constructors), executed by
engine.convformer.ConvFormerRT on sm_90a kernels.  The nn.Modules are parameter containers created in the reference's
order (identical seeded init and state_dict keys); ``forward`` hands the batch to the runtime.
"""
import numpy as np
import torch.nn as nn

from ...engine.convformer import ConvFormerRT
from ...engine.runtime import RuntimeModule

__all__ = ['convformer_s18', 'convformer_s36', 'convformer_m36', 'convformer_b36']


class Downsampling(nn.Module):

    def __init__(self, inplanes, planes, kernel_size, stride=1, padding=0, pre_norm=False, post_norm=False):
        super().__init__()
        self.conv = nn.Conv2d(inplanes, planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=True)
        self.pre_norm = nn.BatchNorm2d(inplanes) if pre_norm else nn.Identity()
        self.post_norm = nn.BatchNorm2d(planes) if post_norm else nn.Identity()


class SepConv(nn.Module):

    def __init__(self, inplanes, kernel_size=7, padding=3, expand_ratio=2):
        super().__init__()
        middle_planes = int(expand_ratio * inplanes)
        self.pwconv1 = nn.Linear(inplanes, middle_planes, bias=False)
        self.act1 = nn.ReLU(inplace=True)
        self.dwconv = nn.Conv2d(middle_planes, middle_planes, kernel_size=kernel_size, padding=padding, groups=middle_planes,
                                bias=False)
        self.act2 = nn.Identity()
        self.pwconv2 = nn.Linear(middle_planes, inplanes, bias=False)


class Mlp(nn.Module):

    def __init__(self, inplanes, mlp_ratio=4, dropout_prob=0.):
        super().__init__()
        hidden_planes = int(mlp_ratio * inplanes)
        self.fc1 = nn.Linear(inplanes, hidden_planes, bias=False)
        self.act = nn.ReLU(inplace=True)
        self.drop1 = nn.Dropout(dropout_prob)
        self.fc2 = nn.Linear(hidden_planes, inplanes, bias=False)
        self.drop2 = nn.Dropout(dropout_prob)


class DropPathBlock(nn.Module):

    def __init__(self, drop_path_prob=0., scale_by_keep=True):
        super().__init__()
        assert drop_path_prob >= 0.
        self.drop_path_prob = drop_path_prob
        self.keep_path_prob = 1 - drop_path_prob
        self.scale_by_keep = scale_by_keep


class MetaFormerBlock(nn.Module):

    def __init__(self, inplanes, dropout_prob=0., drop_path_prob=0.):
        super().__init__()
        self.norm1 = nn.BatchNorm2d(inplanes)
        self.token_mixer = SepConv(inplanes=inplanes, kernel_size=7, padding=3, expand_ratio=2)
        self.norm2 = nn.BatchNorm2d(inplanes)
        self.mlp = Mlp(inplanes=inplanes, mlp_ratio=4, dropout_prob=dropout_prob)
        self.drop_path = DropPathBlock(drop_path_prob) if drop_path_prob > 0. else nn.Identity()


class MetaFormer(RuntimeModule):

    def __init__(self, inplanes=3, embedding_planes=[64, 128, 320, 512], block_nums=[2, 2, 6, 2], dropout_prob=0.,
                 drop_path_prob=0., num_classes=1000, use_gradient_checkpoint=False):
        super().__init__()
        assert len(embedding_planes) == len(block_nums)
        if dropout_prob > 0.:
            raise NotImplementedError('ConvFormer dropout_prob > 0 is not implemented by the H100 runtime (0 in every shipped config)')
        self.block_nums = block_nums
        self.num_classes = num_classes
        self.use_gradient_checkpoint = use_gradient_checkpoint
        planes = [inplanes] + embedding_planes
        self.downsample_layers = nn.ModuleList([
            Downsampling(planes[i], planes[i + 1], kernel_size=7, stride=4, padding=2, pre_norm=False, post_norm=True) if i == 0 else
            Downsampling(planes[i], planes[i + 1], kernel_size=3, stride=2, padding=1, pre_norm=True, post_norm=False)
            for i in range(len(block_nums))])
        rates = [x for x in np.linspace(0, drop_path_prob, sum(block_nums))]
        stages, cur = [], 0
        for i in range(len(block_nums)):
            stages.append(nn.Sequential(*[MetaFormerBlock(inplanes=embedding_planes[i], dropout_prob=dropout_prob,
                                                          drop_path_prob=rates[cur + j]) for j in range(block_nums[i])]))
            cur += block_nums[i]
        self.stages = nn.ModuleList(stages)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.head = nn.Linear(embedding_planes[3], num_classes)
        for m in self.modules():  # convformer.py:231-238
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def _build_runtime(self):
        return ConvFormerRT(self)

    def forward(self, x):
        return self._run(x.float())


def _metaformer(block_nums, embedding_planes, **kwargs):
    return MetaFormer(block_nums=block_nums, embedding_planes=embedding_planes, **kwargs)


def convformer_s18(**kwargs):
    return _metaformer(block_nums=[3, 3, 9, 3], embedding_planes=[64, 128, 320, 512], **kwargs)


def convformer_s36(**kwargs):
    return _metaformer(block_nums=[3, 12, 18, 3], embedding_planes=[64, 128, 320, 512], **kwargs)


def convformer_m36(**kwargs):
    return _metaformer(block_nums=[3, 12, 18, 3], embedding_planes=[96, 192, 384, 576], **kwargs)


def convformer_b36(**kwargs):
    return _metaformer(block_nums=[3, 12, 18, 3], embedding_planes=[128, 256, 512, 768], **kwargs)
