"""Weight gradients of few-filter layers computed as dW^T (saicv_wgrad_transposed): the conv weight gradient with the
im2col patches as an MN-major operand A, and the stem's linear weight gradient with its operands swapped.

Both orientations reduce the same k-blocks over the same splits, so the gradients agree bit for bit with the dW
orientation; that one is reproduced here by an explicit im2col and the (untransposed) linear weight gradient.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _bf(*shape, scale=1.0, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(*shape, device='cuda', generator=g) * scale).to(torch.bfloat16)


CASES = [
    # n, h, c, k, r, transposed
    (4, 56, 64, 64, 3, True),      # ResNet-50 layer1 conv2
    (4, 56, 64, 64, 1, False),     # layer1 block 1 conv1: 64 x 64, both orientations pad alike: stays dW
    (4, 56, 256, 64, 1, True),     # layer1 blocks 2-3 conv1
    (32, 56, 64, 64, 3, True),     # 100352 pixels
    (3, 9, 64, 64, 3, True),       # 243 pixels: a partial reduction block
    (4, 28, 128, 128, 3, False),   # stays dW
]


@pytest.mark.parametrize('n,h,c,k,r,tr', CASES)
def test_conv_wgrad_orientations_agree(n, h, c, k, r, tr):
    ops = _ops()
    pad = r // 2
    x = _bf(n, h, h, c, seed=1)
    dy = _bf(n, h, h, k, scale=(n * h * h) ** -0.5, seed=2)
    cs = ops.make_conv_shape(n, h, h, c, k, r, r, 1, pad)
    ncols = r * r * c
    assert ops.wgrad_transposed(k, ncols) == tr
    part = ops.conv_wgrad(dy, x, cs)
    assert tuple(part.shape[1:]) == ((ncols, k) if tr else (k, ncols))
    dw = torch.empty(k, c, r, r, device='cuda')
    ops.finish_conv_wgrad(part, dw, ncols)
    cols, _, _ = ops.im2col_nhwc(x, r, 1, pad)
    ref_part = ops.linear_wgrad(dy.view(-1, k), cols)          # dW orientation, same splits
    assert ref_part.shape[0] == part.shape[0]
    ref = torch.empty_like(dw)
    ops.finish_conv_wgrad(ref_part, ref, ncols)
    assert torch.equal(dw, ref), f'max diff {(dw - ref).abs().max().item():.3g}'
    want = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), dw.shape, dy.float().permute(0, 3, 1, 2),
                                       padding=pad)
    assert torch.allclose(dw, want, rtol=1e-3, atol=1e-3)
    # gradient accumulation: both layouts add their splits, in order, to what the buffer holds
    start = torch.randn_like(dw)
    acc, acc_ref = start.clone(), start.clone()
    ops.finish_conv_wgrad(part, acc, ncols, accumulate=True)
    ops.finish_conv_wgrad(ref_part, acc_ref, ncols, accumulate=True)
    assert torch.equal(acc, acc_ref)
    assert not torch.equal(acc, dw)


def test_stem_wgrad_transposed_equals_dw():
    """ResNet stem: dW [64, 192] of the explicit-im2col linear weight gradient, as dW^T over the same splits."""
    ops = _ops()
    k, c, r, kpad = 64, 3, 7, ops.stem_kpad(3, 7, 7)
    rows = 2 * 112 * 112
    cols = _bf(rows, kpad, seed=3)
    dy = _bf(rows, k, scale=rows ** -0.5, seed=4)
    assert ops.wgrad_transposed(k, kpad)
    a = ops.linear_wgrad(dy, cols)
    b = ops.linear_wgrad(dy, cols, transposed=True)
    assert a.shape[0] == b.shape[0] and tuple(b.shape[1:]) == (kpad, k)
    dw_a = torch.empty(k, c, r, r, device='cuda')
    dw_b = torch.empty_like(dw_a)
    ops.finish_conv_wgrad(a, dw_a, kpad, order=ops.ORDER_CRS)
    ops.finish_conv_wgrad(b, dw_b, kpad, order=ops.ORDER_CRS)
    assert torch.equal(dw_a, dw_b), f'max diff {(dw_a - dw_b).abs().max().item():.3g}'
