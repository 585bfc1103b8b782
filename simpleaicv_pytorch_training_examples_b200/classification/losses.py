"""Loss tails of the classification step (SURVEY.md §8 a7): fp32 cross entropy on the logits.

Same class names and call signature as SimpleAICV/classification/losses.py:14-28 (CELoss) and
:78-91 (OneHotLabelCELoss).  They stay plain torch: [B, num_classes] fp32 work is negligible
next to the backbone and is not a kernel target; its gradient feeds our backward through
the autograd node of engine.runtime.

SemanticSoftmaxLoss (:94-140, ImageNet-21K semantic-tree training) runs on kernels instead: the reference's version is
~14 small torch kernels per tree level in the forward and as many in the backward, fed by a host-side label conversion
(classification/semantic.py, csrc/capi_loss.cu).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .semantic import SemanticOutputs

__all__ = ['CELoss', 'OneHotLabelCELoss', 'SemanticSoftmaxLoss']


class CELoss(nn.Module):
    """Mean cross entropy over integer labels, computed in fp32."""

    def forward(self, pred, label):
        return F.cross_entropy(pred.float(), label, reduction='mean')


class OneHotLabelCELoss(nn.Module):
    """Mean cross entropy against one-hot / soft labels, computed in fp32."""

    def forward(self, pred, label):
        logp = F.log_softmax(pred.float(), dim=-1)
        return -(label * logp).sum(dim=-1).mean()


class _SemanticSoftmax(torch.autograd.Function):
    """(logits [B, N], semantic labels int64 [B, L]) -> the scalar loss; one kernel pass forward, one backward."""

    @staticmethod
    def forward(ctx, logits, labels, tables, factors, smoothing):
        loss, lse = ops.semantic_softmax_fwd(logits, labels, tables.level_cols, tables.level_off, factors, smoothing)
        ctx.save_for_backward(logits, labels, lse)
        ctx.tables, ctx.factors, ctx.smoothing = tables, factors, smoothing
        return loss

    @staticmethod
    def backward(ctx, grad):
        logits, labels, lse = ctx.saved_tensors
        t = ctx.tables
        dl = ops.semantic_softmax_bwd(logits, labels, t.col_level, t.level_cols, t.level_off, ctx.factors, lse,
                                      grad.float().contiguous(), ctx.smoothing)
        return dl, None, None, None, None


class SemanticSoftmaxLoss(nn.Module):
    """losses.py:94-140 of the reference: per tree level l, label-smoothed cross entropy over the level's classes (rows
    without a label at that level contribute 0 but count in the batch mean), summed over the levels with weight
    normalization_factor_list[l].  Takes the SemanticOutputs of SemanticTree.convert_outputs_to_semantic_outputs and the
    int64 [B, L] labels of convert_single_labels_to_semantic_labels.  CUDA tensors only: there is no CPU fallback."""

    def __init__(self, normalization_factor_list, smoothing):
        super().__init__()
        self.normalization_factor_list = normalization_factor_list
        self.smoothing = float(smoothing)
        # copied to the device once (with .cuda() or at the first call), not per step
        self.register_buffer('factors', torch.as_tensor(normalization_factor_list).reshape(-1).float().clone(), persistent=False)

    def forward(self, semantic_outputs, semantic_labels):
        if not isinstance(semantic_outputs, SemanticOutputs):
            raise TypeError('SemanticSoftmaxLoss takes the SemanticOutputs of SemanticTree.convert_outputs_to_semantic_outputs '
                            '(classification/semantic.py), not a list of per-level slices')
        logits = semantic_outputs.logits
        if not logits.is_cuda:
            raise RuntimeError('SemanticSoftmaxLoss runs on H100 kernels only; move the logits to the GPU (no CPU fallback exists)')
        if logits.dtype not in (torch.float32, torch.bfloat16):
            logits = logits.float()
        logits = logits.contiguous()
        labels = semantic_labels.long().contiguous()
        levels = len(semantic_outputs)
        if labels.shape != (logits.shape[0], levels):
            raise ValueError(f'semantic labels {tuple(labels.shape)} do not match {logits.shape[0]} rows x {levels} levels')
        if self.factors.numel() < levels:
            raise ValueError(f'{self.factors.numel()} normalisation factors for {levels} levels')
        if self.factors.device != logits.device:
            self.factors = self.factors.to(logits.device)
        tables = semantic_outputs.tree.tables(logits.device)
        return _SemanticSoftmax.apply(logits, labels, tables, self.factors, self.smoothing)
