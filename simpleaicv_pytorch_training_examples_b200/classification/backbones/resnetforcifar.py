"""CIFAR ResNets (3x3 stride-1 stem, no max-pool) with the reference's constructor surface
(SimpleAICV/classification/backbones/resnetforcifar.py:27-125), on the H100 runtime."""
from .resnet import BasicBlock, Bottleneck, ConvBnActBlock, _init_like_reference, _ResNetBase

__all__ = ['resnet18cifar', 'resnet34cifar', 'resnet50cifar', 'resnet101cifar', 'resnet152cifar']


class ResNetCifar(_ResNetBase):

    def __init__(self, block, layer_nums, inplanes=64, num_classes=100):
        super().__init__()
        self.num_classes = num_classes
        self.conv1 = ConvBnActBlock(3, inplanes, kernel_size=3, stride=1, padding=1)
        self._build_stages(block, layer_nums, inplanes)
        _init_like_reference(self)


def _resnetcifar(block, layers, inplanes, **kwargs):
    return ResNetCifar(block, layers, inplanes, **kwargs)


def resnet18cifar(**kwargs):
    return _resnetcifar(BasicBlock, [2, 2, 2, 2], 64, **kwargs)


def resnet34cifar(**kwargs):
    return _resnetcifar(BasicBlock, [3, 4, 6, 3], 64, **kwargs)


def resnet50cifar(**kwargs):
    return _resnetcifar(Bottleneck, [3, 4, 6, 3], 64, **kwargs)


def resnet101cifar(**kwargs):
    return _resnetcifar(Bottleneck, [3, 4, 23, 3], 64, **kwargs)


def resnet152cifar(**kwargs):
    return _resnetcifar(Bottleneck, [3, 8, 36, 3], 64, **kwargs)
