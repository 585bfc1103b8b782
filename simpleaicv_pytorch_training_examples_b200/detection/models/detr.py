"""DETR with the reference's constructor surface and state_dict layout (SimpleAICV/detection/models/detr.py:44-90
TransformerEncoderLayer, :93-180 TransformerDecoderLayer, :183-270 DETRTransformer, :273-364 DETR, :367-399
constructors), executed by engine.detr.DetrRT on sm_90a kernels: ResNet body on the conv/BN engine, every Linear on
the wgmma GEMM engine, attention (head size 32, additive key bias in an extra score column) on the wgmma attention
kernels, post-LayerNorm / dropout / head packing in csrc/capi_detr.cu.

The nn.Modules are parameter containers created in the reference's order (identical seeded initialisation and
``state_dict()`` keys); ``forward`` hands the batch to the runtime.  Two behaviours of the reference are kept on
purpose: the transformer receives ``masks.float()``, i.e. nn.MultiheadAttention ADDS +1 to the logits of padded keys
instead of excluding them (detr.py:333-346), and the dropout probability is the constructor constant 0.1.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import backbones
from .backbones.detr_resnet import PositionEmbeddingBlock
from .head import DETRClsRegHead
from ...engine.detr import DetrRT, run_detr

__all__ = ['resnet18_detr', 'resnet34_detr', 'resnet50_detr', 'resnet101_detr', 'resnet152_detr']


class ActivationBlock(nn.Module):

    def __init__(self, act_type='relu'):
        super().__init__()
        assert act_type == 'relu', 'the H100 runtime implements the ReLU feed-forward DETR builds'
        self.act = nn.ReLU(inplace=True)


class TransformerEncoderLayer(nn.Module):

    def __init__(self, hidden_planes, head_nums, feedforward_ratio=4, dropout_prob=0.1, act_type='relu'):
        super().__init__()
        self.attention = nn.MultiheadAttention(hidden_planes, head_nums, dropout=dropout_prob)
        self.linear1 = nn.Linear(hidden_planes, int(hidden_planes * feedforward_ratio))
        self.linear2 = nn.Linear(int(hidden_planes * feedforward_ratio), hidden_planes)
        self.norm1 = nn.LayerNorm(hidden_planes)
        self.norm2 = nn.LayerNorm(hidden_planes)
        self.act = ActivationBlock(act_type)
        self.dropout = nn.Dropout(dropout_prob)


class TransformerDecoderLayer(nn.Module):

    def __init__(self, hidden_planes, head_nums, feedforward_ratio=4, dropout_prob=0.1, act_type='relu'):
        super().__init__()
        self.attention = nn.MultiheadAttention(hidden_planes, head_nums, dropout=dropout_prob)
        self.multihead_attention = nn.MultiheadAttention(hidden_planes, head_nums, dropout=dropout_prob)
        self.linear1 = nn.Linear(hidden_planes, int(hidden_planes * feedforward_ratio))
        self.linear2 = nn.Linear(int(hidden_planes * feedforward_ratio), hidden_planes)
        self.norm1 = nn.LayerNorm(hidden_planes)
        self.norm2 = nn.LayerNorm(hidden_planes)
        self.norm3 = nn.LayerNorm(hidden_planes)
        self.activation = ActivationBlock(act_type)
        self.dropout = nn.Dropout(dropout_prob)


class DETRTransformer(nn.Module):

    def __init__(self, inplanes=256, head_nums=8, feedforward_ratio=4, encoder_layer_nums=6, decoder_layer_nums=6,
                 dropout_prob=0.1, act_type='relu'):
        super().__init__()
        self.inplanes, self.head_nums, self.feedforward_ratio = inplanes, head_nums, feedforward_ratio
        self.encoder_layer_nums, self.decoder_layer_nums = encoder_layer_nums, decoder_layer_nums
        self.dropout_prob, self.act_type = dropout_prob, act_type
        assert inplanes // head_nums == 32, 'the attention kernels are built for DETR\'s head size 32'
        self.encoder_blocks = nn.ModuleList([
            TransformerEncoderLayer(inplanes, head_nums, feedforward_ratio=feedforward_ratio, dropout_prob=dropout_prob,
                                    act_type=act_type) for _ in range(encoder_layer_nums)])
        self.decoder_blocks = nn.ModuleList([
            TransformerDecoderLayer(inplanes, head_nums, feedforward_ratio=feedforward_ratio, dropout_prob=dropout_prob,
                                    act_type=act_type) for _ in range(decoder_layer_nums)])
        self.decoder_norm = nn.LayerNorm(inplanes)
        for m in self.parameters():
            if m.dim() > 1:
                nn.init.xavier_uniform_(m)


class DETR(nn.Module):

    def __init__(self, backbone_type, backbone_pretrained_path='', hidden_inplanes=256, query_nums=100, num_classes=80,
                 use_gradient_checkpoint=False):
        super().__init__()
        self.hidden_inplanes, self.query_nums, self.num_classes = hidden_inplanes, query_nums, num_classes
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.backbone = backbones.__dict__[backbone_type](**{'pretrained_path': backbone_pretrained_path,
                                                             'use_gradient_checkpoint': use_gradient_checkpoint})
        self.position_embedding = PositionEmbeddingBlock(inplanes=hidden_inplanes // 2, temperature=10000, eps=1e-6)
        self.proj_conv = nn.Conv2d(self.backbone.out_channels[-1], hidden_inplanes, kernel_size=1, stride=1, padding=0, bias=True)
        self.transformer = DETRTransformer(inplanes=hidden_inplanes, head_nums=8, feedforward_ratio=4, encoder_layer_nums=6,
                                           decoder_layer_nums=6, dropout_prob=0.1, act_type='relu')
        self.query_embed = nn.Embedding(query_nums, hidden_inplanes)
        self.head = DETRClsRegHead(hidden_inplanes, num_classes + 1, num_layers=3)

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            rt = DetrRT(self)
            self.__dict__['_rt'] = rt  # not a submodule / not in state_dict
        return rt

    def grad_sink(self):
        return self._runtime().sink

    def forward(self, inputs, masks):
        """inputs fp32 [B, 3, H, W]; masks bool [B, H, W] (True = padding).  Returns [cls_outputs [6, B, Q, classes + 1],
        reg_outputs [6, B, Q, 4]] like the reference (detr.py:309-364)."""
        assert masks is not None
        if not inputs.is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU (no CPU fallback exists)')
        fh, fw = _feature_size(inputs.shape[2]), _feature_size(inputs.shape[3])
        fm = F.interpolate(masks.float().unsqueeze(1), size=[fh, fw]).to(torch.bool).squeeze(1)
        pos = self.position_embedding(fm).flatten(2).transpose(1, 2).reshape(-1, self.hidden_inplanes).contiguous()
        key_bias = fm.flatten(1).float().reshape(-1).contiguous()        # float key_padding_mask: +1 on padded keys
        cls, reg = run_detr(self._runtime(), inputs.float(), pos, key_bias, self.training)
        return [cls, reg.float().sigmoid()]


def _feature_size(n):
    """Spatial size of C5 for an input side n: 7x7/2 pad 3, 3x3/2 pad 1 max pool, then three stride-2 stages."""
    n = (n + 2 * 3 - 7) // 2 + 1
    n = (n + 2 * 1 - 3) // 2 + 1
    for _ in range(3):
        n = (n + 2 * 1 - 3) // 2 + 1      # (3x3 pad 1 or 1x1 pad 0 at stride 2 give the same size)
    return n


def _detr(backbone_type, backbone_pretrained_path, **kwargs):
    return DETR(backbone_type, backbone_pretrained_path=backbone_pretrained_path, **kwargs)


def resnet18_detr(backbone_pretrained_path='', **kwargs):
    return _detr('detr_resnet18backbone', backbone_pretrained_path=backbone_pretrained_path, **kwargs)


def resnet34_detr(backbone_pretrained_path='', **kwargs):
    return _detr('detr_resnet34backbone', backbone_pretrained_path=backbone_pretrained_path, **kwargs)


def resnet50_detr(backbone_pretrained_path='', **kwargs):
    return _detr('detr_resnet50backbone', backbone_pretrained_path=backbone_pretrained_path, **kwargs)


def resnet101_detr(backbone_pretrained_path='', **kwargs):
    return _detr('detr_resnet101backbone', backbone_pretrained_path=backbone_pretrained_path, **kwargs)


def resnet152_detr(backbone_pretrained_path='', **kwargs):
    return _detr('detr_resnet152backbone', backbone_pretrained_path=backbone_pretrained_path, **kwargs)
