"""Oracle: the Mixup / CutMix + RandomErasing tail of the ImageNet recipes in float32 on CPU, from the draws a
classification.common.MixupEraseRecord holds.  TEST INFRASTRUCTURE — see oracle/__init__.py.

Restates, from the reference, with torch CPU float32 operations in the reference's order:
- TorchMeanStdNormalize (SimpleAICV/classification/common.py:228-248): ToTensor's float(u8).div(255), Normalize's
  sub_(mean).div_(std), permuted back to [H, W, 3];
- RandomErasing.erase (:614-642) for mode='pixel' and one rectangle: the float noise assigned into the float32 image;
- MixupCutmixClassificationCollater.__call__ (mixupcutmixclassificationcollator.py:140-167): stack, permute to
  [B, 3, H, W]; _mix_batch (:269-284): CutMix copies the box from the flipped batch, Mixup is
  x.mul_(lam).add_(x.flip(0).mul_(1 - lam)); mixup_label (:13-31): one-hots filled with off / on, y1 * lam + y2 * (1 - lam).
"""
import torch

MIX_NONE, MIX_MIXUP, MIX_CUTMIX = 0, 1, 2


def normalize_erase(image_u8, mean, std, rect, noise):
    """One sample: uint8 [H, W, 3] -> float32 [H, W, 3] after TorchMeanStdNormalize and the erase rectangle."""
    t = image_u8.permute(2, 0, 1).contiguous().to(torch.float32).div(255)
    t = t.sub_(torch.tensor(mean, dtype=torch.float32).view(3, 1, 1)).div_(torch.tensor(std, dtype=torch.float32).view(3, 1, 1))
    t = t.permute(1, 2, 0)
    top, left, h, w = (int(v) for v in rect)
    if h > 0 and w > 0:
        t[top:top + h, left:left + w, :] = noise.view(h, w, 3)
    return t


def apply(images_u8, labels, record, mean, std):
    """images_u8 uint8 [B, H, W, 3], labels int64 [B], record: MixupEraseRecord -> (fp32 [B, 3, H, W], fp32 [B, classes])."""
    samples = []
    for b in range(images_u8.shape[0]):
        h, w = int(record.rects[b, 2]), int(record.rects[b, 3])
        off = int(record.offsets[b])
        samples.append(normalize_erase(images_u8[b], mean, std, record.rects[b], record.noise[off:off + h * w * 3]))
    x = torch.stack(samples).permute(0, 3, 1, 2)
    lam = record.lam
    if record.mode == MIX_CUTMIX:
        yl, yh, xl, xh = record.box
        x[:, :, yl:yh, xl:xh] = x.flip(0)[:, :, yl:yh, xl:xh]
    elif record.mode == MIX_MIXUP:
        x_flipped = x.flip(0).mul_(1. - lam)
        x.mul_(lam).add_(x_flipped)
    n, c = labels.shape[0], record.num_classes
    y1 = torch.full((n, c), record.off_value).scatter_(1, labels.view(-1, 1), record.on_value)
    y2 = torch.full((n, c), record.off_value).scatter_(1, labels.flip(0).view(-1, 1), record.on_value)
    return x.contiguous(), y1 * lam + y2 * (1. - lam)
