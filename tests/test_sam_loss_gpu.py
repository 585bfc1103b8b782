"""SAMLoss on the H100 kernels (csrc/capi_loss.cu) against the reference's formulas restated in plain fp32 torch
(interactive_segmentation/losses.py:11-198; tests/golden/make_sam_loss_golden.py runs the reference itself and commits
its outputs for the same seeded inputs): the three loss terms, the best-mask selection (integer indices) and the
gradients w.r.t. the mask logits and the IoU predictions."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk', os.path.join(HERE, 'golden', 'make_sam_loss_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


def _reference_terms(x, t, alpha, gamma, thr):
    """focal / dice / gt_iou [B, M] exactly as losses.py:126-198 computes them (fp32 torch)."""
    b = x.shape[0]
    t = t.expand_as(x).float()
    x = x.float()
    bce = F.binary_cross_entropy_with_logits(x, t, reduction='none')
    p = torch.sigmoid(x)
    pt = p * t + (1 - p) * (1 - t)
    focal = ((alpha * t + (1 - alpha) * (1 - t)) * torch.pow(1. - pt, gamma) * bce).flatten(2).mean(-1) / b
    pf, tf = p.flatten(2), t.flatten(2)
    dice = (1. - (2. * (pf * tf).sum(-1) + 1) / (pf.sum(-1) + tf.sum(-1) + 1)) / b
    xi, ti = (x > thr).flatten(2), (t > thr).flatten(2)
    gt = ((xi & ti).sum(-1).float() / (xi | ti).sum(-1).float().clamp(min=1e-6)).clamp(0., 1.)
    return focal, dice, gt


@pytest.mark.parametrize('B,M,H,W,dtype,gamma', [(2, 4, 64, 64, torch.float32, 2), (3, 1, 32, 48, torch.float32, 2),
                                               (2, 4, 128, 128, torch.bfloat16, 2), (2, 3, 64, 64, torch.float32, 1.5)])
def test_mask_terms_and_gradients_match_torch(B, M, H, W, dtype, gamma):
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.losses import _MaskTerms
    g = torch.Generator().manual_seed(B * 100 + M)
    x = (torch.randn(B, M, H, W, generator=g) * 3).to(dtype)
    t = (torch.rand(B, 1, H, W, generator=g) > 0.6).float()
    xr = x.float().clone().requires_grad_(True)
    f_r, d_r, gt_r = _reference_terms(xr, t, 0.25, gamma, 0.)
    wf, wd = torch.randn(B, M, generator=g), torch.randn(B, M, generator=g)
    ((f_r * wf).sum() + (d_r * wd).sum()).backward()
    xc = x.detach().clone().cuda().requires_grad_(True)
    f, d, gt = _MaskTerms.apply(xc, t.cuda(), 0.25, float(gamma), 0.)
    torch.testing.assert_close(f.cpu(), f_r.detach(), rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(d.cpu(), d_r.detach(), rtol=1e-4, atol=1e-7)
    assert torch.equal(gt.cpu(), gt_r)                               # counts: exact
    ((f * wf.cuda()).sum() + (d * wd.cuda()).sum()).backward()
    rel = ((xc.grad.float().cpu() - xr.grad).norm() / xr.grad.norm()).item()
    assert rel < (1e-2 if dtype == torch.bfloat16 else 1e-4), rel


def test_sam_loss_reproduces_reference_fixture():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.losses import SAMLoss
    fix = torch.load(os.path.join(HERE, 'golden', 'sam_loss_b3.ptl'), weights_only=False)
    for supervise_all in (True, False):
        masks, ious, targets = mk.make_inputs()
        masks = [m.cuda().requires_grad_(True) for m in masks]
        ious = [i.cuda().requires_grad_(True) for i in ious]
        out = SAMLoss(supervise_all_iou=supervise_all)((masks, ious), targets.cuda())
        ref = fix[supervise_all]
        assert list(out) == list(ref['losses'])
        for k, v in ref['losses'].items():
            torch.testing.assert_close(out[k].cpu(), v, rtol=2e-5, atol=1e-7)
        sum(out.values()).backward()
        for m, n in zip(masks, ref['dmask_norm']):
            torch.testing.assert_close(m.grad.norm().cpu(), n, rtol=1e-4, atol=1e-9)
        for i, gi in zip(ious, ref['diou']):
            torch.testing.assert_close(i.grad.cpu(), gi, rtol=1e-4, atol=1e-8)
    with pytest.raises(RuntimeError):
        SAMLoss()(([torch.zeros(1, 4, 8, 8)], [torch.zeros(1, 4)]), torch.zeros(1, 1, 8, 8))
