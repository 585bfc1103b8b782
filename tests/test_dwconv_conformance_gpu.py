"""Conformance of the VAN / ConvFormer depthwise-convolution, gating, layer-scale residual and NHWC im2col kernels
(capi_van.cu) and of the DINOv3 SwiGLU kernels (capi_dinov3.cu) against a float64 reference, and their bit-identity
invariants.

Reference.  Every check computes the exact result in float64 on the GPU from the same bf16 / fp32 values the kernel
read (a product of a bf16 and an fp32 value, or of two bf16 values, is exact in float64).  The depthwise references
are written tap by tap on a zero-padded copy of the input; test_dwconv_reference_matches_torch checks them against
torch's float64 conv2d and its autograd input and weight gradients.

Allowances are derived from the operation, never fitted to measured errors.  u = 2^-24 is one fp32 rounding, and
gamma(m) = m u / (1 - m u) bounds m chained roundings.
  * dwconv_fwd: the exact value is v = bias + sum x w over the in-image taps.  The kernel starts from the fp32 bias
    and chains at most K^2 fmaf calls in (r, s) order, so its fp32 value is within gamma(K^2) (|bias| + sum |x w|) of v.
    ReLU is 1-Lipschitz.  flip=True (the data gradient) is checked against the float64 input gradient of the same
    convolution with the same allowance and no bias.
  * dwconv_dgrad_masked: the same allowance where mask > 0; where mask <= 0 (including -0.0) the output is +0, checked
    as raw bits.
  * dwconv_wgrad: each thread chains ceil(ppb / 32) fmaf over its pixels of the block (ppb = ceil(npix / nblk), nblk
    from saicv_dwconv_wgrad_blocks), the block adds its 32 thread sums in order, and the fold adds the nblk block
    partials in order: depth d = ceil(ppb / 32) + 32 + nblk (+1 with accumulate).  fp32 output within
    (d + 1) u (sum |dy x| + |previous dw|).
  * mul_bf16: a product of two bf16 values is exact in fp32, so the output must be rne_bf16(a b), bit for bit.
  * gate_bwd: one fmaf, so the fp32 value is within u |v| of v = dg c1 + dlk, then rounded to bf16; where p1 <= 0 the
    output is +0 (raw bits).
  * ls_residual_fwd: out = fmaf(s ls, b', x) with b' = branch (+ shortcut).  s ls and the shortcut add round before
    the fmaf: the product carries gamma(1 + shortcut) |s ls b'|, and the fmaf rounds once more.
  * ls_residual_bwd: dy = bf16((s ls) g) carries gamma(2) |v| before its bf16 rounding.  dls sums the terms
    (s g) b' with their own gamma(1 + shortcut) through the slab reduction: per-thread chain ceil(rpb / ty) + the
    ty_count rows of the block + the nblk partial rows of reduce_partials (+1 with accumulate), with (ty, rpb, nblk)
    from the Python mirror of capi_van.cu slab; allowance (d + 1 + 1 + shortcut) u sum |terms| + (d + 1) u |prev|.
  * swiglu: silu(a) = a / (1 + expf(-a)).  expf is accurate to 2 ulp (CUDA C Programming Guide), i.e. 4u relative,
    plus 2^-148 absolute for a subnormal result; __fadd_rn and __fdiv_rn round once each.  Every fp32 rounding is
    taken as u relative plus 2^-150 absolute (gradual underflow: sg and the products below it reach the fp32
    subnormal range near a = -88).  Where e^-a exceeds the fp32 range (a <= -89 in bf16) expf returns +inf and the
    kernels return 0 for silu and for da, as torch's fp32 silu does; those elements are checked to be 0 and kept out
    of the interval check (there |silu(a)| < 2^-120).  The stored h = bf16(silu(a)) lies in the bf16 interval of
    that allowance.  da = bf16((ds sg) (1 + a (1 - sg))) with ds = bf16(dh b), itself a correctly rounded product, so
    the float64 reference starts from rne_bf16(dh b); the allowance carries sg's through 1 - sg (which is large
    relative to 1 - sg near sg = 1), a (1 - sg), 1 + ..., ds sg and the final product, one rounding each.  h and db
    are products of two bf16 values (b or dh times the stored bf16 silu), so given the stored silu they are bit-exact.
  * im2col_nhwc is bit-exact against a float64 unfold, including its zero padding.  col2im_nhwc adds at most
    ceil(k / s)^2 bf16 terms in (r, s) order from 0: fp32 within gamma(ceil(k / s)^2) sum |terms|, then bf16.
  * A bf16 output shows its fp32 error only where the exact value lies within B of a bf16 rounding boundary, so
    families whose fp32 value is exact or a few roundings from it (gate_bwd, col2im, silu) can report a share of 0,
    as the bit-exact ones do.

Launch geometry.  Python mirrors of grid_1d (host_util.cu), saicv_dwconv_wgrad_blocks and
ppb; every shape list asserts that it runs a grid-stride loop more than once, and the weight-gradient list that it
has nblk = 132 with a ragged last block.

Invariants (raw bits): outputs and partial workspaces are filled with NaN before each launch, so an unwritten
element or a folded stale partial fails, and two consecutive launches give identical outputs.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conformance import NAN, U, call, check, every_bf16, exact, nan, rand, randn, rne_bf16, rnd, same, van_slab
from conformance import report  # noqa: F401  (autouse: this module's allowance report)

from simpleaicv_pytorch_training_examples_b200 import _lib, ops

pytestmark = pytest.mark.gpu

ETA = 2.0 ** -150           # one fp32 rounding in the subnormal range, absolute
EXP_REL = 4 * U             # expf: 2 ulp
EXP_ABS = 2.0 ** -148       # expf: 2 ulp of a subnormal result
FP32_OVF = 2.0 ** 128 * (1 - 2.0 ** -25)    # an fp32 rounding of a value at or above this gives +inf
BF16 = torch.bfloat16


def _gamma(m):
    return m * U / (1 - m * U)


def _zero_bits(what, out, dead):
    """Raw +0 where `dead`."""
    bad = int((out.view(torch.int16)[dead] != 0).sum())
    assert bad == 0, f'{what}: {bad}/{int(dead.sum())} masked elements are not +0'


# ------------------------------------------------------------------ launch geometry mirrors
def _grid_1d(items, per_block=256, cap=132 * 16):
    """host_util.cu grid_1d."""
    return max(1, min(-(-items // per_block), cap))


def _loops(items, per_block, blocks):
    """Trips of the grid-stride loop for the first thread."""
    return -(-items // (per_block * blocks))


def _wgrad_blocks(npix):
    """capi_van.cu saicv_dwconv_wgrad_blocks."""
    return max(1, min(-(-npix // 256), 132))


def _ppb(npix):
    return -(-npix // _wgrad_blocks(npix))


def _dw_loops(n, h, w):
    npix = n * h * w
    return _loops(npix, 32, _grid_1d(npix, 32, 132 * 8))


# ------------------------------------------------------------------ shape lists
KD = [(3, 1), (5, 1), (7, 1), (7, 3)]
DW_C = [8, 32, 72, 160, 1152, 1536]
DW_MAPS = [(1, 1), (2, 3), (5, 9), (7, 7), (14, 14), (56, 56)]
# every (k, dil) x C x map, up to 4 images; then VAN-B0 stage 1 at batch 64 (the LKA 5x5 and 7x7 dilation-3
# convolutions) and ConvFormer-S18 stage 1 (SepConv 7x7 on 2 x 64 channels) at batch 32
DW_FWD = [(max(1, min(4, 200000 // (h * w * c))), h, w, c, k, dil) for k, dil in KD for c in DW_C for h, w in DW_MAPS]
DW_FWD += [(64, 56, 56, 32, 5, 1), (64, 56, 56, 32, 7, 3), (32, 56, 56, 128, 7, 1)]
assert any(_dw_loops(n, h, w) > 1 for n, h, w, *_ in DW_FWD)
assert any(h != w for _, h, w, *_ in DW_FWD)
assert any(c == 8 for *_, c, _, _ in DW_FWD) and (7, 7, 7, 3) in [(h, w, k, dil) for _, h, w, _, k, dil in DW_FWD]

DW_MASKED = [(2, 1, 1, 8), (3, 2, 3, 72), (2, 5, 9, 160), (4, 7, 7, 1536), (8, 14, 14, 640), (3, 13, 29, 64),
             (32, 56, 56, 128)]
assert any(_dw_loops(n, h, w) > 1 for n, h, w, _ in DW_MASKED)
assert any(h != w for _, h, w, _ in DW_MASKED)

DW_WGRAD = [(2, 1, 1, 8, 7, 3), (3, 2, 3, 32, 3, 1), (2, 5, 9, 72, 5, 1), (4, 7, 7, 1536, 7, 3), (5, 13, 7, 160, 7, 1),
            (3, 17, 40, 1152, 3, 1), (2, 96, 176, 8, 5, 1), (16, 56, 56, 256, 3, 1), (64, 56, 56, 32, 5, 1),
            (64, 56, 56, 32, 7, 3), (32, 56, 56, 128, 7, 1)]


def _ragged(npix):
    return _wgrad_blocks(npix) * _ppb(npix) != npix


assert any(_wgrad_blocks(n * h * w) == 132 and _ragged(n * h * w) for n, h, w, *_ in DW_WGRAD)
assert any(_wgrad_blocks(n * h * w) == 132 and not _ragged(n * h * w) for n, h, w, *_ in DW_WGRAD)
assert any(h != w for _, h, w, *_ in DW_WGRAD)

GATE = [(1, 8), (294, 96), (4 * 3136, 64), (64 * 3136, 256)]      # the last: VAN-B0 stage-1 gating at batch 64
assert any(_loops(r * c // 8, 256, _grid_1d(r * c // 8)) > 1 for r, c in GATE)

# (rows, C, rows per drop-path scale): a single row, ViT-style token rows, VAN stage-1 at batch 64, and slab
# reductions that use all 264 partial rows (40000 x 384 with a short last block, 8448 x 1536 with a full one)
LS = [(1, 8, 1), (147, 1536, 49), (1570, 384, 785), (50176, 8, 3136), (40000, 384, 800), (2113, 1536, 197),
      (8448, 1536, 264), (64 * 3136, 32, 3136)]
assert any(_loops(r * c // 8, 256, _grid_1d(r * c // 8)) > 1 for r, c, _ in LS)
assert any(van_slab(r, c)[2] == 264 for r, c, _ in LS)

SWIGLU_N = [8, 4104, 6291456]
assert any(_loops(n // 8, 256, _grid_1d(n // 8)) > 1 for n in SWIGLU_N)

# (n, h, w, c, k, stride, pad): VAN-B0 patch embeddings of stages 2-4 (3x3 s2 p1) at batch 64 / 16, maps where
# (h + 2p - k) % s != 0, h != w, the 7x7 s4 p3 stem shape with 8 and 24 channels, and a 1x1 map
IM2COL = [(64, 56, 56, 32, 3, 2, 1), (16, 28, 28, 64, 3, 2, 1), (8, 14, 14, 160, 3, 2, 1), (2, 10, 10, 32, 3, 2, 1),
          (3, 13, 10, 16, 3, 2, 1), (2, 224, 224, 8, 7, 4, 3), (1, 30, 17, 24, 7, 4, 3), (1, 1, 1, 8, 3, 2, 1)]


def _out_size(h, k, s, p):
    return (h + 2 * p - k) // s + 1


assert any(_loops(n * _out_size(h, k, s, p) * _out_size(w, k, s, p) * k * k * c // 8, 256,
                  _grid_1d(n * _out_size(h, k, s, p) * _out_size(w, k, s, p) * k * k * c // 8)) > 1
           for n, h, w, c, k, s, p in IM2COL)
assert any(_loops(n * h * w * c // 8, 256, _grid_1d(n * h * w * c // 8)) > 1 for n, h, w, c, *_ in IM2COL)
assert any((h + 2 * p - k) % s for _, h, _, _, k, s, p in IM2COL)


def test_launch_geometry_mirrors_match_the_library():
    """The mirrors against the host functions the library exports: saicv_dwconv_wgrad_blocks, and the block count of
    capi_van.cu slab (saicv_bn_generic_partial_rows), which ls_residual_bwd shares."""
    lib = _lib.load()
    for npix in [1, 255, 256, 257, 33535, 33536, 33537, 200704, 100352]:
        assert lib.saicv_dwconv_wgrad_blocks(npix) == _wgrad_blocks(npix), npix
    for rows, c, _ in LS:
        assert lib.saicv_bn_generic_partial_rows(rows, c) == van_slab(rows, c)[2], (rows, c)


# ------------------------------------------------------------------ depthwise references
def _dw_ref(x, w, k, dil, flip=False):
    """float64 (sum of products over the in-image taps, sum of their absolute values), [N, H, W, C].
    flip=False: y[h, w] = sum_rs x[h + r dil - pad, w + s dil - pad] w[r, s] (the 'same' convolution);
    flip=True: its input gradient, dx[h, w] = sum_rs dy[h - r dil + pad, w - s dil + pad] w[r, s]."""
    n, h, wd, c = x.shape
    pad = dil * (k - 1) // 2
    xp = F.pad(x.double(), (0, 0, pad, pad, pad, pad))
    w64 = w.double().reshape(c, k, k)
    v = torch.zeros(n, h, wd, c, dtype=torch.float64, device=x.device)
    a = torch.zeros_like(v)
    for r in range(k):
        for s in range(k):
            oh, ow = (2 * pad - r * dil, 2 * pad - s * dil) if flip else (r * dil, s * dil)
            t = xp[:, oh:oh + h, ow:ow + wd, :] * w64[:, r, s]
            v += t
            a += t.abs()
    return v, a


def _dw_wgrad_ref(dy, x, k, dil):
    """float64 dw[c][r][s] = sum_pix dy[pix] x[pix + tap offset] and the sum of the absolute terms, [C, 1, K, K]."""
    n, h, wd, c = x.shape
    pad = dil * (k - 1) // 2
    xp = F.pad(x.double(), (0, 0, pad, pad, pad, pad))
    g = dy.double()
    v = torch.empty(c, k, k, dtype=torch.float64, device=x.device)
    a = torch.empty_like(v)
    for r in range(k):
        for s in range(k):
            t = g * xp[:, r * dil:r * dil + h, s * dil:s * dil + wd, :]
            v[:, r, s] = t.sum((0, 1, 2))
            a[:, r, s] = t.abs().sum((0, 1, 2))
    return v.view(c, 1, k, k), a.view(c, 1, k, k)


def test_dwconv_reference_matches_torch():
    """The tap-by-tap references above against torch's float64 conv2d, its input gradient and its weight gradient."""
    for n, h, w, c, k, dil in [(2, 5, 9, 8, 7, 3), (1, 6, 4, 16, 5, 1), (2, 3, 2, 8, 3, 1)]:
        x = randn(n, c, h, w, seed=1).double().requires_grad_(True)
        wt = randn(c, 1, k, k, seed=2).double().requires_grad_(True)
        dy = randn(n, c, h, w, seed=3).double()
        y = F.conv2d(x, wt, None, 1, dil * (k - 1) // 2, dil, c)
        y.backward(dy)
        nhwc = lambda t: t.detach().permute(0, 2, 3, 1).contiguous()
        torch.testing.assert_close(_dw_ref(nhwc(x), wt.detach(), k, dil)[0], nhwc(y), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(_dw_ref(nhwc(dy), wt.detach(), k, dil, flip=True)[0], nhwc(x.grad), rtol=1e-12,
                                   atol=1e-12)
        torch.testing.assert_close(_dw_wgrad_ref(nhwc(dy), nhwc(x), k, dil)[0], wt.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------ depthwise convolution
def _dwconv(x, w, bias, k, dil, relu, flip):
    n, h, wd, c = x.shape
    y = torch.full_like(x, NAN)
    call('saicv_dwconv_fwd', x, w, bias, y, n, h, wd, c, k, dil, int(relu), int(flip))
    return y


def _dw_case(n, h, w, c, k, seed):
    x = randn(n, h, w, c, seed=seed).to(BF16)
    wt = randn(c, 1, k, k, seed=seed + 1) / k
    bias = randn(c, seed=seed + 2) * 0.5
    return x, wt, bias


@pytest.mark.parametrize('n,h,w,c,k,dil', DW_FWD)
def test_dwconv_fwd_conforms(n, h, w, c, k, dil):
    """saicv_dwconv_fwd with bias and without, ReLU on and off, and flip=True against the input gradient."""
    seed = 1000 + 7 * n + 131 * h + 17 * w + c + 1000 * k + dil
    x, wt, bias = _dw_case(n, h, w, c, k, seed)
    what = f'dwconv {n}x{h}x{w}x{c} k{k} d{dil}'
    v, a = _dw_ref(x, wt, k, dil)
    b64 = bias.double()
    g = _gamma(k * k)
    for use_bias in (True, False):
        vb = v + b64 if use_bias else v
        ab = g * (a + b64.abs()) if use_bias else g * a
        for relu in (False, True):
            y = _dwconv(x, wt, bias if use_bias else None, k, dil, relu, False)
            tag = f'{what}{" bias" if use_bias else ""}{" relu" if relu else ""}'
            check('dwconv fwd', tag, y, vb.clamp_min(0) if relu else vb, ab)
            same(f'{tag} on a second launch', y, _dwconv(x, wt, bias if use_bias else None, k, dil, relu, False))
        del vb, ab
    del v, a
    dy = randn(n, h, w, c, seed=seed + 3).to(BF16)
    v, a = _dw_ref(dy, wt, k, dil, flip=True)
    dx = _dwconv(dy, wt, None, k, dil, False, True)
    check('dwconv fwd flip (dgrad)', f'{what} flip', dx, v, g * a)
    same(f'{what} flip on a second launch', dx, _dwconv(dy, wt, None, k, dil, False, True))


def _dgrad_masked(dy, w, mask):
    n, h, wd, c = dy.shape
    dx = torch.full_like(dy, NAN)
    call('saicv_dwconv_dgrad_masked', dy, w, mask, dx, n, h, wd, c, 7)
    return dx


@pytest.mark.parametrize('n,h,w,c', DW_MASKED)
def test_dwconv_dgrad_masked_conforms(n, h, w, c):
    """saicv_dwconv_dgrad_masked (ConvFormer's 7x7 data gradient through the ReLU in front of the conv).  The mask
    is a ReLU output with its lower half of rows and every third channel zero, -0.0 on a checkerboard of the zeros,
    and a few negative values."""
    seed = 2000 + 7 * n + 131 * h + 17 * w + c
    dy, wt, _ = _dw_case(n, h, w, c, 7, seed)
    m = randn(n, h, w, c, seed=seed + 5).clamp_min(0)
    m[:, (h + 1) // 2:] = 0
    m[..., ::3] = 0
    checker = ((torch.arange(h, device='cuda')[:, None] + torch.arange(w, device='cuda')[None, :]) % 2 == 0)
    m = torch.where((m == 0) & checker[None, :, :, None], torch.tensor(-0.0, device='cuda'), m)
    m[..., 1::7] = -rand(n, h, w, len(range(1, c, 7)), seed=seed + 6)
    mask = m.to(BF16)
    live = mask.double() > 0
    assert live.any() and (~live).any() and bool((mask.view(torch.int16) == -32768).any())   # -0.0 present
    what = f'dwconv dgrad masked {n}x{h}x{w}x{c}'
    v, a = _dw_ref(dy, wt, 7, 1, flip=True)
    dx = _dgrad_masked(dy, wt, mask)
    check('dwconv dgrad masked', what, dx[live], v[live], _gamma(49) * a[live])
    _zero_bits(what, dx, ~live)
    same(f'{what} on a second launch', dx, _dgrad_masked(dy, wt, mask))


def _wgrad(dy, x, k, dil, dw, accumulate):
    n, h, wd, c = x.shape
    npix = n * h * wd
    nblk = _lib.load().saicv_dwconv_wgrad_blocks(npix)
    assert nblk == _wgrad_blocks(npix)
    partial = nan(nblk * k * k * c)
    call('saicv_dwconv_wgrad', dy, x, partial, dw, n, h, wd, c, k, dil, int(accumulate))
    return dw


@pytest.mark.parametrize('n,h,w,c,k,dil', DW_WGRAD)
def test_dwconv_wgrad_conforms(n, h, w, c, k, dil):
    """saicv_dwconv_wgrad into a NaN-filled dw and accumulated onto a previous dw, with a NaN-filled partial buffer of
    nblk k^2 C floats."""
    seed = 3000 + 7 * n + 131 * h + 17 * w + c + 1000 * k + dil
    x = randn(n, h, w, c, seed=seed).to(BF16)
    dy = randn(n, h, w, c, seed=seed + 1).to(BF16)
    npix = n * h * w
    nblk, ppb = _wgrad_blocks(npix), _ppb(npix)
    d = -(-ppb // 32) + 32 + nblk
    what = f'dwconv wgrad {n}x{h}x{w}x{c} k{k} d{dil} (nblk {nblk}, ppb {ppb})'
    v, a = _dw_wgrad_ref(dy, x, k, dil)
    dw = _wgrad(dy, x, k, dil, nan(c, 1, k, k), False)
    check('dwconv wgrad', what, dw, v, (d + 1) * U * a)
    same(f'{what} on a second launch', dw, _wgrad(dy, x, k, dil, nan(c, 1, k, k), False))
    prev = randn(c, 1, k, k, seed=seed + 2) * a.mean().float().sqrt()
    dw2 = _wgrad(dy, x, k, dil, prev.clone(), True)
    v2 = v + prev.double()
    check('dwconv wgrad', f'{what} accumulate', dw2, v2, (d + 2) * U * (a + prev.double().abs()))
    same(f'{what} accumulate on a second launch', dw2, _wgrad(dy, x, k, dil, prev.clone(), True))


# ------------------------------------------------------------------ gating
def _mul(a, b):
    out = torch.full_like(a, NAN)
    call('saicv_mul_bf16', a, b, out, a.numel())
    return out


def _gate_bwd(dg, c1, dlk, p1):
    out = torch.full_like(dg, NAN)
    call('saicv_gate_bwd', dg, c1, dlk, p1, out, dg.numel())
    return out


@pytest.mark.parametrize('rows,c', GATE)
def test_mul_and_gate_bwd_conform(rows, c):
    """saicv_mul_bf16 bit for bit against rne_bf16(a b); saicv_gate_bwd against dg c1 + dlk where p1 > 0 and +0 where
    p1 <= 0 (p1 a ReLU output with -0.0 on every fifth zero)."""
    seed = 4000 + rows + c
    a, b, dlk = (randn(rows, c, seed=seed + i).to(BF16) for i in range(3))
    p = randn(rows, c, seed=seed + 3).clamp_min(0)
    p.view(-1)[::5] = torch.where(p.view(-1)[::5] == 0, torch.tensor(-0.0, device='cuda'), p.view(-1)[::5])
    p1 = p.to(BF16)
    del p
    what = f'gating {rows}x{c}'
    out = _mul(a, b)
    exact('mul_bf16', f'{what} mul_bf16', out, rne_bf16(a.double() * b.double()).to(BF16))
    same(f'{what} mul_bf16 on a second launch', out, _mul(a, b))
    del out
    live = p1.double() > 0
    out = _gate_bwd(a, b, dlk, p1)
    v = a.double()[live] * b.double()[live] + dlk.double()[live]
    check('gate_bwd', f'{what} gate_bwd', out[live], v, U * v.abs())
    del v
    _zero_bits(f'{what} gate_bwd', out, ~live)
    same(f'{what} gate_bwd on a second launch', out, _gate_bwd(a, b, dlk, p1))


# ------------------------------------------------------------------ layer-scale residual
def _ls_fwd(x, br, sc, ls, rs, rps):
    rows, c = br.shape
    out = nan(rows, c)
    call('saicv_ls_residual_fwd', x, int(x.dtype == torch.float32), br, sc, ls, rs, rps, out, rows, c)
    return out


def _ls_bwd(dxn, br, sc, ls, rs, rps, dls, accumulate):
    rows, c = br.shape
    dy = torch.full((rows, c), NAN, device='cuda', dtype=BF16)
    ws = ops.partial_ws(dxn.device, 2 * c)
    ws.fill_(NAN)
    call('saicv_ls_residual_bwd', dxn, br, sc, ls, rs, rps, dy, ws, dls, rows, c, int(accumulate))
    return dy


@pytest.mark.parametrize('rows,c,rps', LS)
@pytest.mark.parametrize('shortcut', [False, True])
def test_ls_residual_conforms(rows, c, rps, shortcut):
    """saicv_ls_residual_fwd / _bwd: x fp32 or bf16 (alternating over the cases), drop-path row scales 0 or
    float32(1 / 0.9) per rps rows (none on every third case), dls written and accumulated."""
    i = LS.index((rows, c, rps)) * 2 + int(shortcut)
    seed = 5000 + 10 * i
    x_f32 = i % 2 == 0
    x = randn(rows, c, seed=seed) * 2
    x = x if x_f32 else x.to(BF16)
    br = randn(rows, c, seed=seed + 1).to(BF16)
    sc = randn(rows, c, seed=seed + 2).to(BF16) if shortcut else None
    ls = (rand(c, seed=seed + 3) * 2 - 1) * 0.5
    nsc = -(-rows // rps)
    keep = rand(nsc, seed=seed + 4) > 0.3
    keep[0] = True
    rs = None if i % 3 == 2 else torch.where(keep, torch.tensor(1 / 0.9, device='cuda'), torch.tensor(0.0, device='cuda'))
    dxn = randn(rows, c, seed=seed + 5)
    what = f'ls_residual rows {rows} c {c} x {"f32" if x_f32 else "bf16"}{" shortcut" if shortcut else ""}' \
           f'{"" if rs is None else f" drop-path/{rps}"}'
    s = rs.double().repeat_interleave(rps)[:rows, None] if rs is not None else 1.0
    b = br.double() + (sc.double() if shortcut else 0.0)
    k = 1 + int(shortcut)                     # roundings before the fmaf / inside a dls term
    # forward
    P = s * ls.double() * b
    v = x.double() + P
    out = _ls_fwd(x, br, sc, ls, rs, rps)
    check('ls_residual fwd', what, out, v, rnd(v, _gamma(k) * P.abs()))
    same(f'{what} fwd on a second launch', out, _ls_fwd(x, br, sc, ls, rs, rps))
    del P, v, out
    # backward
    g = dxn.double()
    vd = s * ls.double() * g
    dls = nan(c)
    dy = _ls_bwd(dxn, br, sc, ls, rs, rps, dls, False)
    check('ls_residual bwd dy', f'{what} dy', dy, vd, _gamma(2) * vd.abs())
    del vd
    t = s * g * b
    st, sa = t.sum(0), t.abs().sum(0)
    del t
    ty, rpb, nblk = van_slab(rows, c)
    d = -(-rpb // ty) + ty + nblk
    check('ls_residual bwd dls', f'{what} dls (slab {nblk} x {rpb} rows)', dls, st, (d + 1 + k) * U * sa)
    prev = randn(c, seed=seed + 6) * sa.float().mean()
    dls2 = prev.clone()
    dy2 = _ls_bwd(dxn, br, sc, ls, rs, rps, dls2, True)
    same(f'{what} dy (accumulate call)', dy2, dy)
    v2 = prev.double() + st
    check('ls_residual bwd dls', f'{what} dls accumulate', dls2, v2,
          (d + 2 + k) * U * sa + (d + 2) * U * prev.double().abs())
    dls3 = nan(c)
    same(f'{what} dy on a second launch', _ls_bwd(dxn, br, sc, ls, rs, rps, dls3, False), dy)
    same(f'{what} dls on a second launch', dls3, dls)


# ------------------------------------------------------------------ SwiGLU
def _fl(v, a):
    """Allowance after one fp32 rounding (gradual underflow included) of a value within a of v."""
    return a + U * (v.abs() + a) + ETA


def _fmul(x, ax, y, ay):
    v = x * y
    return v, _fl(v, x.abs() * ay + y.abs() * ax + ax * ay)


def _fdiv(x, ax, d, ad):
    """x / d for d > ad >= 0."""
    v = x / d
    return v, _fl(v, (ax + v.abs() * ad) / (d - ad))


def _swiglu_ref(a64, ds):
    """Exact silu(a) and ds silu'(a), with the allowances of the kernels' fp32 values, for a where expf does not
    overflow.  ds: the exact float64 value of the kernel's bf16 ds."""
    e = torch.exp(-a64)
    den, a_den = 1 + e, _fl(1 + e, EXP_REL * e + EXP_ABS)            # __fadd_rn(1, expf(-a))
    silu, a_silu = _fdiv(a64, 0.0, den, a_den)                       # __fdiv_rn(a, .)
    sg, a_sg = _fdiv(torch.ones_like(a64), 0.0, den, a_den)          # __fdiv_rn(1, .)
    m, a_m = 1 - sg, _fl(1 - sg, a_sg)                               # __fsub_rn(1, sg)
    p, a_p = _fmul(a64, 0.0, m, a_m)                                 # __fmul_rn(a, 1 - sg)
    q, a_q = 1 + p, _fl(1 + p, a_p)                                  # __fadd_rn(1, .)
    t, a_t = _fmul(ds, 0.0, sg, a_sg)                                # __fmul_rn(ds, sg)
    da, a_da = _fmul(t, a_t, q, a_q)                                 # __fmul_rn(., .)
    return silu, a_silu, da, a_da


def _overflow(a64):
    """(expf(-a) certainly +inf, expf(-a) certainly finite); a 2-ulp expf is certain on both sides for bf16 a."""
    e = torch.exp(-a64)
    inf = e * (1 - EXP_REL) >= FP32_OVF
    fin = e * (1 + EXP_REL) < FP32_OVF
    assert bool((inf | fin).all()), 'a bf16 input lies where a 2-ulp expf may or may not overflow'
    return inf, fin


def _swiglu_fwd(a, b):
    out = torch.full_like(a, NAN)
    call('saicv_swiglu_fwd', a, b, out, a.numel())
    return out


def _swiglu_bwd(dh, a, b):
    da, db = torch.full_like(a, NAN), torch.full_like(a, NAN)
    call('saicv_swiglu_bwd', dh, a, b, da, db, a.numel())
    return da, db


def _check_swiglu(what, a, h, da, ds):
    """h = bf16(silu(a)) (b = 1) and da against the float64 reference from ds."""
    a64 = a.double()
    inf, fin = _overflow(a64)
    silu, a_silu, g, a_g = _swiglu_ref(a64[fin], ds[fin])
    if h is not None:
        check('swiglu silu', f'{what} silu', h[fin], silu, a_silu)
        assert bool((h[inf].double() == 0).all()), f'{what}: silu is not 0 where expf(-a) overflows'
    check('swiglu da', f'{what} da', da[fin], g, a_g)
    assert bool((da[inf].double() == 0).all()), f'{what}: da is not 0 where expf(-a) overflows'


def test_swiglu_on_every_bf16_input():
    """Every finite bf16 a with b = 1 and dh = 1: h is the stored bf16(silu(a)), db equals it, and da = silu'(a)."""
    a = every_bf16(256).view(-1)
    one = torch.ones_like(a)
    h = _swiglu_fwd(a, one)
    da, db = _swiglu_bwd(one, a, one)
    what = 'swiglu on every bf16 a'
    _check_swiglu(what, a, h, da, torch.ones_like(a, dtype=torch.float64))
    exact('swiglu db', f'{what} db (dh = 1)', db, h)
    same(f'{what} h on a second launch', h, _swiglu_fwd(a, one))
    da2, db2 = _swiglu_bwd(one, a, one)
    same(f'{what} da on a second launch', da2, da)
    same(f'{what} db on a second launch', db2, db)


@pytest.mark.parametrize('n', SWIGLU_N)
def test_swiglu_random_b_dh_conforms(n):
    """Random a (4 randn), b and dh: h = rne(silu_b b) and db = rne(dh silu_b) bit for bit given the stored bf16
    silu_b = swiglu_fwd(a, 1), and da against ds silu'(a) with ds = rne_bf16(dh b)."""
    a = (randn(n, seed=6000 + n) * 4).to(BF16)
    b = randn(n, seed=6001 + n).to(BF16)
    dh = randn(n, seed=6002 + n).to(BF16)
    what = f'swiglu n {n}'
    s = _swiglu_fwd(a, torch.ones_like(a)).double()
    h = _swiglu_fwd(a, b)
    exact('swiglu h', f'{what} h', h, rne_bf16(s * b.double()).to(BF16))
    da, db = _swiglu_bwd(dh, a, b)
    exact('swiglu db', f'{what} db', db, rne_bf16(dh.double() * s).to(BF16))
    _check_swiglu(what, a, None, da, rne_bf16(dh.double() * b.double()))
    same(f'{what} h on a second launch', h, _swiglu_fwd(a, b))
    da2, db2 = _swiglu_bwd(dh, a, b)
    same(f'{what} da on a second launch', da2, da)
    same(f'{what} db on a second launch', db2, db)


# ------------------------------------------------------------------ NHWC im2col / col2im
def _im2col(x, k, st, pad):
    n, h, w, c = x.shape
    P, Q = _out_size(h, k, st, pad), _out_size(w, k, st, pad)
    cols = torch.full((n * P * Q, k * k * c), NAN, device='cuda', dtype=BF16)
    call('saicv_im2col_nhwc', x, cols, n, h, w, c, k, st, pad)
    return cols


def _col2im(dcols, n, h, w, c, k, st, pad):
    dx = torch.full((n, h, w, c), NAN, device='cuda', dtype=BF16)
    call('saicv_col2im_nhwc', dcols, dx, n, h, w, c, k, st, pad)
    return dx


@pytest.mark.parametrize('n,h,w,c,k,st,pad', IM2COL)
def test_im2col_col2im_nhwc_conform(n, h, w, c, k, st, pad):
    """saicv_im2col_nhwc bit for bit against F.unfold in float64 (rows (n, p, q), columns (r, s, c)), and
    saicv_col2im_nhwc against F.fold in float64."""
    seed = 7000 + n + h + 3 * w + c + k
    P, Q = _out_size(h, k, st, pad), _out_size(w, k, st, pad)
    x = randn(n, h, w, c, seed=seed).to(BF16)
    what = f'im2col {n}x{h}x{w}x{c} k{k} s{st} p{pad}'
    ref = F.unfold(x.double().permute(0, 3, 1, 2), k, padding=pad, stride=st)          # [n, c k^2, P Q]
    ref = ref.view(n, c, k * k, P * Q).permute(0, 3, 2, 1).reshape(n * P * Q, k * k * c)
    cols = _im2col(x, k, st, pad)
    exact('im2col_nhwc', what, cols, ref.to(BF16))
    same(f'{what} on a second launch', cols, _im2col(x, k, st, pad))
    del ref, cols
    dcols = randn(n * P * Q, k * k * c, seed=seed + 1).to(BF16)

    def fold(t):
        t = t.view(n, P * Q, k * k, c).permute(0, 3, 2, 1).reshape(n, c * k * k, P * Q)
        return F.fold(t, (h, w), k, padding=pad, stride=st).permute(0, 2, 3, 1)

    v, a = fold(dcols.double()), fold(dcols.double().abs())
    dx = _col2im(dcols, n, h, w, c, k, st, pad)
    what = f'col2im {n}x{h}x{w}x{c} k{k} s{st} p{pad}'
    check('col2im_nhwc', what, dx, v, _gamma(math.ceil(k / st) ** 2) * a)
    same(f'{what} on a second launch', dx, _col2im(dcols, n, h, w, c, k, st, pad))
