"""Loss tails of the classification step (SURVEY.md §8 a7): fp32 cross entropy on the logits.

Same class names and call signature as SimpleAICV/classification/losses.py:14-28 (CELoss) and
:78-91 (OneHotLabelCELoss).  They stay plain torch: [B, num_classes] fp32 work is negligible
next to the backbone and is not a kernel target; its gradient feeds our backward through
the autograd node of engine.runtime.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ['CELoss', 'OneHotLabelCELoss']


class CELoss(nn.Module):
    """Mean cross entropy over integer labels, computed in fp32."""

    def forward(self, pred, label):
        return F.cross_entropy(pred.float(), label, reduction='mean')


class OneHotLabelCELoss(nn.Module):
    """Mean cross entropy against one-hot / soft labels, computed in fp32."""

    def forward(self, pred, label):
        logp = F.log_softmax(pred.float(), dim=-1)
        return -(label * logp).sum(dim=-1).mean()
