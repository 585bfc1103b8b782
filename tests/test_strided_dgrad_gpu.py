"""Data gradient of 3x3 stride-2 convolutions by output phase (saicv_conv_dgrad with stride 2).

The phase path reduces, for every dx pixel, exactly the non-zero taps the stride-1 kernel reduces over the
zero-upsampled dy, in the same order, so the two agree bit for bit (torch.equal: -0.0 == 0.0, the sign of an exact
zero may differ).  Both are also checked against torch's fp32 conv2d_input within bf16 tolerance.
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


def _case(n, h, w, c, k):
    ops = _ops()
    wt = _bf(k, c, 3, 3, scale=(9 * c) ** -0.5, seed=8).float()
    wb = torch.empty(k, 9 * c, device='cuda', dtype=torch.bfloat16)
    ops.prep_conv_weight(wt.contiguous(), wb, 9 * c)
    cs = ops.make_conv_shape(n, h, w, c, k, 3, 3, 2, 1)
    P, Q = ops.conv_out_size(h, 1, 3, 2), ops.conv_out_size(w, 1, 3, 2)
    dy = _bf(n, P, Q, k, seed=9)
    return ops, wt, wb, cs, dy


def _upsampled(ops, dy, wb, cs, add=None):
    u = ops.zero_upsample2(dy, cs.h, cs.w)
    cs1 = ops.make_conv_shape(cs.n, cs.h, cs.w, cs.c, cs.k, 3, 3, 1, 1)
    return ops.conv_dgrad(u, wb, cs1, add=add)


def _torch_ref(wt, dy, cs):
    dy_nchw = dy.float().permute(0, 3, 1, 2)
    return torch.nn.grad.conv2d_input((cs.n, cs.c, cs.h, cs.w), wt, dy_nchw, stride=2, padding=1).permute(0, 2, 3, 1)


def _close(got, ref, what):
    err = (got.float() - ref).abs()
    bad = (err > 2e-2 + 1e-2 * ref.abs()).sum().item()
    assert bad == 0, f'{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}'


PHASE_CASES = [
    (4, 56, 56, 128, 128),     # ResNet-50 layer2 conv2
    (4, 28, 28, 256, 256),     # layer3
    (4, 14, 14, 512, 512),     # layer4
    (32, 56, 56, 128, 128),    # 25088 rows per phase
    (256, 14, 14, 512, 512),   # bs256 layer4: 12544 rows per phase
    (4, 64, 64, 64, 128),      # DarkNet downsampling unit (BN = 64 tiles)
    (3, 10, 10, 64, 64),       # 75 rows per phase: one partial tile
    (2, 26, 18, 128, 64),      # h != w, Q = 9: 14 dy rows per tile
    (1, 256, 256, 64, 64),     # Q = 128: one dy row per tile
]


@pytest.mark.parametrize('n,h,w,c,k', PHASE_CASES)
def test_phase_dgrad_equals_upsampled_path(n, h, w, c, k):
    ops, wt, wb, cs, dy = _case(n, h, w, c, k)
    assert ops.phase_dgrad_ok(cs)
    got = ops.conv_dgrad(dy, wb, cs)
    ref = _upsampled(ops, dy, wb, cs)
    assert torch.equal(got, ref), f'{(got.float() - ref.float()).abs().max().item():.4g}'
    _close(got, _torch_ref(wt, dy, cs), 'phase dgrad vs torch')


def test_phase_dgrad_overwrites_every_pixel():
    """Each of the four phases writes its own pixels: no dx element keeps what the buffer held."""
    ops, wt, wb, cs, dy = _case(3, 28, 28, 128, 128)
    out = torch.full((cs.n, cs.h, cs.w, cs.c), float('nan'), device='cuda', dtype=torch.bfloat16)
    ops.conv_dgrad(dy, wb, cs, out=out)
    assert not out.isnan().any()
    assert torch.equal(out, _upsampled(ops, dy, wb, cs))


@pytest.mark.parametrize('n,h,w,c,k', [(2, 15, 15, 64, 128), (3, 7, 9, 128, 64), (1, 260, 260, 64, 64)])
def test_strided_dgrad_fallback(n, h, w, c, k):
    """Odd sizes and rows wider than a tile go through the zero-upsampled stride-1 path."""
    ops, wt, wb, cs, dy = _case(n, h, w, c, k)
    assert not ops.phase_dgrad_ok(cs)
    got = ops.conv_dgrad(dy, wb, cs)
    assert torch.equal(got, _upsampled(ops, dy, wb, cs))
    _close(got, _torch_ref(wt, dy, cs), 'fallback dgrad vs torch')


def test_strided_dgrad_with_add_falls_back():
    ops, wt, wb, cs, dy = _case(2, 28, 28, 128, 128)
    add = _bf(2, 28, 28, 128, seed=23)
    got = ops.conv_dgrad(dy, wb, cs, add=add)
    assert torch.equal(got, _upsampled(ops, dy, wb, cs, add=add))


def test_phase_dgrad_refuses_add_and_unsupported_shapes():
    from simpleaicv_pytorch_training_examples_b200 import _lib
    ops, wt, wb, cs, dy = _case(2, 28, 28, 128, 128)
    dx = torch.empty(2, 28, 28, 128, device='cuda', dtype=torch.bfloat16)
    add = torch.zeros_like(dx)
    with pytest.raises(RuntimeError, match='add'):
        _lib.call('saicv_conv_dgrad', dy.data_ptr(), wb.data_ptr(), add.data_ptr(), None, dx.data_ptr(), ops.ctypes.byref(cs),
                  None)
    odd = ops.make_conv_shape(2, 27, 27, 128, 128, 3, 3, 2, 1)
    with pytest.raises(RuntimeError, match='even'):
        _lib.call('saicv_conv_dgrad', dy.data_ptr(), wb.data_ptr(), None, None, dx.data_ptr(), ops.ctypes.byref(odd), None)
