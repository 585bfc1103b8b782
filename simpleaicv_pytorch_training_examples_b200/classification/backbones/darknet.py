"""DarknetTiny / Darknet19 / Darknet53 with the reference's constructor surface and state_dict layout
(SimpleAICV/classification/backbones/darknet.py:16-31 ActivationBlock, :34-65 ConvBnActBlock,
:68-113 Darknet19Block, :116-144 Darknet53Block, :147-244 DarknetTiny, :247-320 Darknet19,
:323-432 Darknet53, :435-450 constructors), executed by engine.convnet on sm_90a kernels.

Layers whose channel counts are not multiples of 64 (16/32-channel stacks) run on channel-padded
activations inside the runtime; parameters keep the reference's shapes.  The 2x2 max-pools, the
ZeroPad2d + stride-1 pool of DarknetTiny and Darknet19's biased 1x1-conv classifier are runtime
stages (engine.convnet.MaxPoolRT / ConvHeadRT).
"""
import torch.nn as nn

from ...engine.convnet import ACT_LEAKY, ACT_RELU, ACT_SILU, ConvBN, ConvHeadRT, DarkBlockRT, MaxPoolRT, PlainUnitRT, ResNetRT
from ...engine.runtime import RuntimeModule
from .resnet import _init_like_reference  # same initialisation as the reference's darknet.py:218-225,299-306,397-404

__all__ = ['darknettiny', 'darknet19', 'darknet53']

_ACT = {'relu': ACT_RELU, 'leakyrelu': ACT_LEAKY, 'silu': ACT_SILU}


class ActivationBlock(nn.Module):

    def __init__(self, act_type='leakyrelu', inplace=True):
        super().__init__()
        assert act_type in ['silu', 'relu', 'leakyrelu'], 'Unsupport activation function!'
        if act_type == 'silu':
            self.act = nn.SiLU(inplace=inplace)
        elif act_type == 'relu':
            self.act = nn.ReLU(inplace=inplace)
        else:
            self.act = nn.LeakyReLU(0.1, inplace=inplace)


class ConvBnActBlock(nn.Module):

    def __init__(self, inplanes, planes, kernel_size, stride, padding, groups=1, has_bn=True, has_act=True,
                 act_type='leakyrelu'):
        super().__init__()
        assert groups == 1
        self.layer = nn.Sequential(
            nn.Conv2d(inplanes, planes, kernel_size, stride=stride, padding=padding, groups=groups, bias=not has_bn),
            nn.BatchNorm2d(planes) if has_bn else nn.Sequential(),
            ActivationBlock(act_type=act_type, inplace=True) if has_act else nn.Sequential())


class Darknet19Block(nn.Module):

    def __init__(self, inplanes, planes, layer_num, use_maxpool=False, act_type='leakyrelu'):
        super().__init__()
        self.use_maxpool = use_maxpool
        layers = []
        for i in range(layer_num):
            if i % 2 == 0:
                layers.append(ConvBnActBlock(inplanes, planes, kernel_size=3, stride=1, padding=1, act_type=act_type))
            else:
                layers.append(ConvBnActBlock(planes, inplanes, kernel_size=1, stride=1, padding=0, act_type=act_type))
        self.Darknet19Block = nn.Sequential(*layers)
        if self.use_maxpool:
            self.MaxPool = nn.MaxPool2d(kernel_size=2, stride=2)


class Darknet53Block(nn.Module):

    def __init__(self, inplanes, act_type='leakyrelu'):
        super().__init__()
        squeezed = int(inplanes // 2)
        self.conv = nn.Sequential(
            ConvBnActBlock(inplanes, squeezed, kernel_size=1, stride=1, padding=0, act_type=act_type),
            ConvBnActBlock(squeezed, inplanes, kernel_size=3, stride=1, padding=1, act_type=act_type))


class _DarknetBase(RuntimeModule):

    def forward(self, x):
        return self._run(x.float())


class DarknetTiny(_DarknetBase):

    def __init__(self, act_type='leakyrelu', num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.act_type = act_type
        for i, (cin, cout) in enumerate([(3, 16), (16, 32), (32, 64), (64, 128), (128, 256), (256, 512)]):
            setattr(self, f'conv{i + 1}', ConvBnActBlock(cin, cout, kernel_size=3, stride=1, padding=1, act_type=act_type))
            if i < 5:
                setattr(self, f'maxpool{i + 1}', nn.MaxPool2d(kernel_size=2, stride=2))
        self.zeropad = nn.ZeroPad2d((0, 1, 0, 1))
        self.maxpool6 = nn.MaxPool2d(kernel_size=2, stride=1)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512, self.num_classes)
        _init_like_reference(self)

    def _build_runtime(self):
        act = _ACT[self.act_type]
        stages = [MaxPoolRT(2, 2)]
        for i in range(2, 7):
            stages.append(PlainUnitRT(getattr(self, f'conv{i}'), act))
            if i < 6:
                stages.append(MaxPoolRT(2, 2))
        stages.append(MaxPoolRT(2, 1, pad=0, pad_hi=1, oob_zero=True))   # ZeroPad2d((0,1,0,1)) + MaxPool2d(2, 1)
        return ResNetRT(self, has_maxpool=False, stem=ConvBN(self.conv1, act), blocks=stages)


class Darknet19(_DarknetBase):

    def __init__(self, act_type='leakyrelu', num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.act_type = act_type
        self.layer1 = ConvBnActBlock(3, 32, kernel_size=3, stride=1, padding=1, act_type=act_type)
        self.maxpool1 = nn.MaxPool2d(kernel_size=2, stride=2)
        self.layer2 = Darknet19Block(32, 64, layer_num=1, use_maxpool=True, act_type=act_type)
        self.layer3 = Darknet19Block(64, 128, layer_num=3, use_maxpool=True, act_type=act_type)
        self.layer4 = Darknet19Block(128, 256, layer_num=3, use_maxpool=True, act_type=act_type)
        self.layer5 = Darknet19Block(256, 512, layer_num=5, use_maxpool=True, act_type=act_type)
        self.layer6 = Darknet19Block(512, 1024, layer_num=5, use_maxpool=False, act_type=act_type)
        self.layer7 = ConvBnActBlock(1024, self.num_classes, kernel_size=1, stride=1, padding=0, has_bn=False,
                                     has_act=False, act_type=act_type)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        _init_like_reference(self)

    def _build_runtime(self):
        act = _ACT[self.act_type]
        stages = [MaxPoolRT(2, 2)]
        for i in range(2, 7):
            blk = getattr(self, f'layer{i}')
            stages += [PlainUnitRT(u, act) for u in blk.Darknet19Block]
            if blk.use_maxpool:
                stages.append(MaxPoolRT(2, 2))
        return ResNetRT(self, has_maxpool=False, stem=ConvBN(self.layer1, act), blocks=stages,
                        head=ConvHeadRT(self.layer7.layer[0]))


class Darknet53(_DarknetBase):

    def __init__(self, act_type='leakyrelu', num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.act_type = act_type
        self.conv1 = ConvBnActBlock(3, 32, kernel_size=3, stride=1, padding=1, act_type=act_type)
        widths = [(32, 64, 1), (64, 128, 2), (128, 256, 8), (256, 512, 8), (512, 1024, 4)]
        for i, (cin, cout, nblocks) in enumerate(widths):
            setattr(self, f'conv{i + 2}', ConvBnActBlock(cin, cout, kernel_size=3, stride=2, padding=1, act_type=act_type))
            setattr(self, f'block{i + 1}', nn.Sequential(*[Darknet53Block(cout, act_type=act_type) for _ in range(nblocks)]))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(1024, num_classes)
        _init_like_reference(self)

    def _build_runtime(self):
        act = _ACT[self.act_type]
        stages = []
        for i in range(5):
            stages.append(PlainUnitRT(getattr(self, f'conv{i + 2}'), act))
            stages += [DarkBlockRT(b, act) for b in getattr(self, f'block{i + 1}')]
        return ResNetRT(self, has_maxpool=False, stem=ConvBN(self.conv1, act), blocks=stages)


def darknettiny(**kwargs):
    return DarknetTiny(**kwargs)


def darknet19(**kwargs):
    return Darknet19(**kwargs)


def darknet53(**kwargs):
    return Darknet53(**kwargs)
