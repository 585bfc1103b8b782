"""Encoder-distillation loss with the reference's interface (SimpleAICV/interactive_segmentation/distill_losses.py:10-23):
fp32 torch on the [B, 256, H/16, W/16] encoder outputs."""
import torch.nn as nn

__all__ = [
    'MSELoss',
]


class MSELoss(nn.Module):

    def __init__(self):
        super().__init__()
        self.loss = nn.MSELoss(reduction='mean')

    def forward(self, tea_preds, stu_preds):
        return {'distill_mse_loss': self.loss(stu_preds, tea_preds)}
