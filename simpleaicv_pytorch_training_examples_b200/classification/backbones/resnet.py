"""ResNet 18/34/50/101/152 with the reference's constructor surface and state_dict layout
(SimpleAICV/classification/backbones/resnet.py:19-48 ConvBnActBlock, :51-97 BasicBlock,
:100-155 Bottleneck, :158-245 ResNet, :254-271 constructors), executed by
engine.convnet.ResNetRT on hand-written sm_90a kernels.

The nn.Modules below are parameter containers: they create the same torch submodules in the same
order as the reference (so seeded initialisation and ``state_dict()`` keys/shapes are identical)
but ``forward`` never calls them; it hands the batch to the runtime.  A CPU tensor raises: there
is no fallback path.
"""
import torch
import torch.nn as nn

from ...engine.convnet import ResNetRT, run_network

__all__ = ['resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152']


class ConvBnActBlock(nn.Module):
    """conv(no bias) -> BatchNorm2d -> ReLU, held as ``layer = Sequential(conv, bn, act)``."""

    def __init__(self, inplanes, planes, kernel_size, stride, padding, groups=1, has_bn=True, has_act=True):
        super().__init__()
        assert groups == 1 and has_bn, 'the H100 runtime implements the conv+BN blocks the ResNets use'
        conv = nn.Conv2d(inplanes, planes, kernel_size, stride=stride, padding=padding, groups=groups, bias=False)
        self.layer = nn.Sequential(conv, nn.BatchNorm2d(planes),
                                   nn.ReLU(inplace=True) if has_act else nn.Sequential())

    def forward(self, x):
        raise RuntimeError('ConvBnActBlock is executed by engine.convnet, call the network instead')


def _cba(cin, cout, k, stride, act):
    return ConvBnActBlock(cin, cout, kernel_size=k, stride=stride, padding=k // 2, has_act=act)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        self.downsample = stride != 1 or inplanes != planes
        self.conv1 = _cba(inplanes, planes, 3, stride, True)
        self.conv2 = _cba(planes, planes, 3, 1, False)
        self.relu = nn.ReLU(inplace=True)
        if self.downsample:
            self.downsample_conv = _cba(inplanes, planes, 1, stride, False)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        self.downsample = stride != 1 or inplanes != planes * 4
        self.conv1 = _cba(inplanes, planes, 1, 1, True)
        self.conv2 = _cba(planes, planes, 3, stride, True)
        self.conv3 = _cba(planes, planes * 4, 1, 1, False)
        self.relu = nn.ReLU(inplace=True)
        if self.downsample:
            self.downsample_conv = _cba(inplanes, planes * 4, 1, stride, False)


def _init_like_reference(model):
    # resnet.py:206-213: kaiming-normal(fan_out) convs, unit BN scale, zero BN shift
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
        elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
            nn.init.constant_(m.weight, 1)
            nn.init.constant_(m.bias, 0)


class _ResNetBase(nn.Module):
    """Shared body: 4 stages of residual blocks, global average pool, fc."""

    def _build_stages(self, block, layer_nums, inplanes):
        self.block = block
        self.layer_nums = layer_nums
        self.inplanes = inplanes
        self.planes = [inplanes, inplanes * 2, inplanes * 4, inplanes * 8]
        self.expansion = block.expansion
        for i, (planes, stride) in enumerate(zip(self.planes, (1, 2, 2, 2))):
            blocks = []
            for j in range(layer_nums[i]):
                blocks.append(block(self.inplanes, planes, stride if j == 0 else 1))
                self.inplanes = planes * self.expansion
            setattr(self, f'layer{i + 1}', nn.Sequential(*blocks))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(self.planes[3] * self.expansion, self.num_classes)

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            rt = ResNetRT(self, has_maxpool=hasattr(self, 'maxpool1'),
                          checkpoint=getattr(self, 'use_gradient_checkpoint', False))
            self.__dict__['_rt'] = rt  # not a submodule / not in state_dict
        return rt

    def grad_sink(self):
        """Where the runtime deposits parameter gradients (used by distributed.B200DataParallel)."""
        return self._runtime().sink

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU '
                               '(no CPU fallback exists)')
        return run_network(self._runtime(), x.float(), self.training)


class ResNet(_ResNetBase):

    def __init__(self, block, layer_nums, inplanes=64, num_classes=1000, use_gradient_checkpoint=False):
        super().__init__()
        self.num_classes = num_classes
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.conv1 = ConvBnActBlock(3, inplanes, kernel_size=7, stride=2, padding=3)
        self.maxpool1 = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self._build_stages(block, layer_nums, inplanes)
        _init_like_reference(self)


def _resnet(block, layers, inplanes, **kwargs):
    return ResNet(block, layers, inplanes, **kwargs)


def resnet18(**kwargs):
    return _resnet(BasicBlock, [2, 2, 2, 2], 64, **kwargs)


def resnet34(**kwargs):
    return _resnet(BasicBlock, [3, 4, 6, 3], 64, **kwargs)


def resnet50(**kwargs):
    return _resnet(Bottleneck, [3, 4, 6, 3], 64, **kwargs)


def resnet101(**kwargs):
    return _resnet(Bottleneck, [3, 4, 23, 3], 64, **kwargs)


def resnet152(**kwargs):
    return _resnet(Bottleneck, [3, 8, 36, 3], 64, **kwargs)
