"""SAMLoss with the reference's interface (SimpleAICV/interactive_segmentation/losses.py:11-198): per prompt iteration
a sigmoid focal loss and a dice loss on the best of the M predicted masks plus an MSE on the predicted IoUs, averaged
over the iterations.  Everything that touches the [B, M, H, W] logits runs in two kernels of libsaicv_b200.so
(csrc/capi_loss.cu): one pass reduces the six per-mask sums the three terms need, one pass writes the logit gradient;
the [B, M]-sized bookkeeping (best-mask selection, weights, the IoU MSE) stays in torch and is differentiated by
autograd.  CUDA tensors only: there is no CPU fallback.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops

__all__ = ['SAMLoss']


class _MaskTerms(torch.autograd.Function):
    """(mask logits [B, M, H, W], targets [B, 1, H, W]) -> focal [B, M], dice [B, M] (each already divided by the batch
    size, like losses.py:126-170) and the thresholded ground-truth IoU [B, M] (no gradient)."""

    @staticmethod
    def forward(ctx, logits, targets, alpha, gamma, thr):
        if not logits.is_cuda:
            raise RuntimeError('SAMLoss runs on H100 kernels only; move the predictions to the GPU (no CPU fallback exists)')
        logits = logits.contiguous()
        if logits.dtype not in (torch.float32, torch.bfloat16):
            logits = logits.float()
        targets = targets.float().contiguous()
        b = logits.shape[0]
        n = logits[0, 0].numel()
        s = ops.sam_loss_sums(logits, targets, alpha, gamma, thr)
        focal = s[..., 0] / (n * b)
        denom = s[..., 2] + s[..., 3] + 1.
        dice = (1. - (2. * s[..., 1] + 1.) / denom) / b
        gt_iou = (s[..., 4] / s[..., 5].clamp(min=1e-6)).clamp(min=0., max=1.)
        ctx.save_for_backward(logits, targets, s)
        ctx.cfg = (alpha, gamma)
        ctx.mark_non_differentiable(gt_iou)
        return focal, dice, gt_iou

    @staticmethod
    def backward(ctx, dfocal, ddice, _):
        logits, targets, s = ctx.saved_tensors
        alpha, gamma = ctx.cfg
        b = logits.shape[0]
        n = logits[0, 0].numel()
        denom = s[..., 2] + s[..., 3] + 1.
        # dice = (1 - (2 S_pt + 1) / D) / b,  dS_pt/dx = sigmoid' t,  dD/dx = sigmoid'
        coef = torch.stack([dfocal / (n * b), ddice * (-2. / (b * denom)), ddice * ((2. * s[..., 1] + 1.) / (b * denom * denom))], dim=-1)
        return ops.sam_loss_bwd(logits, targets, coef.float(), alpha, gamma), None, None, None, None


class SAMLoss(nn.Module):

    def __init__(self, alpha=0.25, gamma=2, focal_loss_weight=20, dice_loss_weight=1, iou_predict_loss_weight=1, supervise_all_iou=True,
                 mask_threshold=0.):
        super().__init__()
        self.alpha, self.gamma = alpha, gamma
        self.focal_loss_weight, self.dice_loss_weight, self.iou_predict_loss_weight = focal_loss_weight, dice_loss_weight, iou_predict_loss_weight
        self.supervise_all_iou = supervise_all_iou
        self.mask_threshold = mask_threshold

    def compute_per_iter_loss(self, mask_preds, iou_preds, targets):
        """(sum over the batch of the best mask's focal loss, of its dice loss, of the IoU-prediction loss), losses.py:78-124."""
        b = mask_preds.shape[0]
        focal, dice, gt_iou = _MaskTerms.apply(mask_preds, targets, float(self.alpha), float(self.gamma), float(self.mask_threshold))
        iou_loss = F.mse_loss(iou_preds.float(), gt_iou, reduction='none') / b
        if focal.shape[1] > 1:
            best = torch.argmin(focal * self.focal_loss_weight + dice * self.dice_loss_weight, dim=-1)
            rows = torch.arange(b, device=focal.device)
            focal, dice = focal[rows, best].unsqueeze(1), dice[rows, best].unsqueeze(1)
            iou_loss = iou_loss.mean(dim=-1, keepdim=True) if self.supervise_all_iou else iou_loss[rows, best].unsqueeze(1)
        return focal.sum(), dice.sum(), iou_loss.sum()

    def forward(self, all_iter_preds, targets):
        """all_iter_preds = (list of mask logits [B, M, H, W], list of IoU predictions [B, M]) over the prompt iterations;
        targets [B, 1, H, W].  Returns {'focal_loss', 'dice_loss', 'iou_predict_loss'} (weighted, averaged over iterations)."""
        masks, ious = all_iter_preds
        assert len(masks) == len(ious)
        focal = dice = iou = 0.
        for m, i in zip(masks, ious):
            f, d, u = self.compute_per_iter_loss(m, i, targets)
            focal, dice, iou = focal + f, dice + d, iou + u
        k = float(len(masks))
        return {'focal_loss': focal / k * self.focal_loss_weight, 'dice_loss': dice / k * self.dice_loss_weight,
                'iou_predict_loss': iou / k * self.iou_predict_loss_weight}
