"""Conformance of the conv operand-layout and gradient-assembly kernels of csrc/capi_elementwise.cu, bit for bit: the
explicit stem im2col, the weight-operand copy, the conv weight-gradient finish, the split-K partial reduction, the
fp32 -> bf16 cast, the bf16 add and the two stride-2 scatters.

Every one of these kernels copies values, rounds once to bf16 (round to nearest even), or adds fp32 values in a fixed
order, so the exact result of every element is known and the bar is bit equality (raw bits: signed zeros count):
  * stem_im2col: cols[n*P*Q][kpad], column (c*R + r)*S8 + s (S8 = S rounded up to 8) holds rne(x[n, c, p*stride - pad + r,
    q*stride - pad + s]); out-of-image taps, columns with s >= S and columns >= C*R*S8 hold +0.0;
  * prep_conv_weight: w_bf16[kp][kpad], order 0 column tap*cp + c, order 1 column (c*R + r)*S8 + s, hold rne(w); every
    other element (filters >= K, channels >= C, the S8 padding, columns past the map) holds +0.0;
  * finish_conv_wgrad: grad = (accumulate ? grad : 0) + partial[0][map] + partial[1][map] + ..., one fp32 add per split in
    ascending order, from [kp][kpad] or dW^T [kpad][kp] partials; every position the map must not read holds NaN, so a
    stray read makes the output non-finite.  It is also checked against float64 with (splits + 1) u sum|terms|;
  * reduce_partials: out = (accumulate ? out : 0) + partial[0] + partial[1] + ..., in ascending order, and its float4
    and scalar paths give identical bits;
  * cast_bf16: every finite or infinite input gives its integer-RNE bf16, a NaN gives a NaN (payload unspecified),
    on the vector path and on the scalar path (n % 8 != 0, misaligned source or destination);
  * add_bf16 / add_strided2: a <- rne(fl32(a + b)), the fp32 sum rounded once more to bf16.  For two bf16 operands this
    double rounding never differs from one rounding of the exact sum: the fp32 sum is exact unless the exponents differ
    by more than 16, and then it lies within 2^-16 of the larger operand, far from any bf16 midpoint.  The cases include
    such gaps, exact cancellations (a + (-a) = +0.0) and -0.0 + -0.0;
  * zero_upsample2: u[n, 2p, 2q] = dy[n, p, q] bit for bit (NaN payloads included), +0.0 elsewhere.
bf16 references are computed by integer RNE on the fp32 bit pattern, (u + 0x7FFF + ((u >> 16) & 1)) >> 16, never by a
cast.  Every input that passes through a rounding carries signed zeros, ties on odd and even bf16 mantissas, fp32
subnormals and values at or above the overflow point (0x7F7F8000 -> inf).  Every output is prefilled with NaN, so an
element the kernel never writes fails.

Two compositions check that the producing and consuming layouts agree, under the GEMM engine's accumulation allowance
(conformance.acc_allowance, test_gemm_conformance_gpu.py) carried through one fp32 rounding per finish add:
  * the stem at the ResNet 7x7/2 and ViT 16/16 geometries: stem_im2col + prep_conv_weight(order 1) + linear_fwd against
    float64 F.conv2d of the bf16-rounded image and weight, and linear_wgrad + finish_conv_wgrad(order 1) against float64
    conv2d_weight (the ResNet stem runs its weight gradient as dW^T, the ViT patch embedding as dW);
  * a channel- and filter-padded conv: conv_wgrad on zero-padded channels, then finish_conv_wgrad(kp, cp), against
    float64 conv2d_weight of the unpadded problem, once as dW^T and once as dW.

The refusals of each C entry return an error and launch nothing.  A 3-channel 64 x 64 / 64 patch is exactly 48 KiB at
one output pixel per block and still runs; a 4-channel one does not fit and is refused.

Largest shares of the allowance, measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: the finish against
float64 65 % (a sequential fp32 sum may use most of it), the stem weight gradient 1.3 %, the padded conv weight gradient
0.9 %, the stem forward 0.5 %; every bit-exact family 0.  The file runs in about 13 s.
"""
import re

import numpy as np
import pytest
import torch
from torch.nn.grad import conv2d_weight
import torch.nn.functional as F

from conformance import M32, U, acc_allowance, call, check, exact, gen, nan, rand, randn, rnd, same
from conformance import report  # noqa: F401  (autouse: this module's allowance report)

from simpleaicv_pytorch_training_examples_b200 import _lib, ops

gpu = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
CAP = 132 * 16 * 256    # items one sweep of grid_1d covers (132 * 16 blocks of 256 threads)

# fp32 bit patterns every rounded input carries
ROUNDING_SPECIALS = [
    0x00000000, 0x80000000,             # +-0
    0x3F808000, 0xBF808000,             # ties on an even bf16 mantissa: stay
    0x3F818000, 0xBF818000,             # ties on an odd bf16 mantissa: round away to the even neighbour
    0x3F807FFF, 0x3F808001,             # either side of a tie
    0x00000001, 0x80000001,             # smallest subnormals: round to +-0
    0x00008000, 0x00018000, 0x80018000,  # subnormal ties
    0x007FFFFF, 0x807FFFFF,             # largest subnormals: round up to the smallest normal
    0x7F7F7FFF, 0xFF7F7FFF,             # just below the overflow point: +-max bf16
    0x7F7F8000, 0xFF7F8000,             # the overflow point: +-inf
    0x7F7FFFFF, 0xFF7FFFFF,             # fp32 max: +-inf
    0x7F800000, 0xFF800000,             # +-inf
]
# bf16 bit patterns of the add inputs
BF16_SPECIALS = [0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x0080, 0x7F7F, 0xFF7F, 0x7F80, 0xFF80, 0x3F80, 0xBF80]


# ------------------------------------------------------------------ references
def _f32_bits(patterns):
    return torch.from_numpy(np.array(patterns, dtype=np.uint32).view(np.int32)).cuda().view(F32)


def _bf16_bits(patterns):
    return torch.from_numpy(np.array(patterns, dtype=np.uint16).view(np.int16)).cuda().view(BF16)


def rne_bits(x):
    """fp32 -> bf16 by integer round-to-nearest-even on the bit pattern (finite and infinite inputs; not NaN)."""
    u = x.contiguous().view(torch.int32).to(torch.int64) & M32
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16).view(BF16)


def fl32_add(a, b):
    """fp32 sum of two fp32 / bf16 tensors, rounded once (the float64 sum of two floats is exact or rounded harmlessly:
    53 >= 2 * 24 + 2)."""
    return (a.double() + b.double()).float()


def _exact_or_nan(family, what, out, v):
    """out (bf16) must be rne_bits(v) wherever v (fp32) is not NaN, and a NaN where it is."""
    bad = torch.isnan(v)
    if bad.any():
        assert torch.isnan(out[bad].float()).all(), f'{what}: a NaN input or sum gave a non-NaN'
    exact(family, what, out[~bad], rne_bits(v[~bad]))


def _sprinkle(x, seed, frac=1 / 16):
    """x (fp32, modified in place) with about `frac` of its elements replaced by ROUNDING_SPECIALS."""
    flat = x.view(-1)
    sel = (rand(flat.numel(), seed=seed) < frac).nonzero().flatten()
    spec = _f32_bits(ROUNDING_SPECIALS)
    flat[sel] = spec[torch.randint(0, spec.numel(), (sel.numel(),), device='cuda', generator=gen(seed + 1))]
    return x


def _wide(*shape, seed=0):
    """fp32 values over 40 binades with full 24-bit mantissas, so every element is rounded."""
    e = torch.randint(-20, 20, shape, device='cuda', generator=gen(seed + 7)).float()
    return randn(*shape, seed=seed) * torch.exp2(e)


def _s8(s):
    return (s + 7) // 8 * 8


def _stem_tile(c, r, s, stride):
    """saicv_stem_im2col's output pixels per block: halved from 32 until the staged patch fits in 40 KB."""
    t = 32
    while t > 1 and c * r * ((t - 1) * stride + s) * 4 > 40 * 1024:
        t >>= 1
    return t


def _stem_ref(x, r, s, stride, pad, kpad):
    n, c, h, w = x.shape
    P, Q = ops.conv_out_size(h, pad, r, stride), ops.conv_out_size(w, pad, s, stride)
    xp = torch.zeros(n, c, h + 2 * pad, w + 2 * pad, device='cuda', dtype=BF16)
    xp[:, :, pad:pad + h, pad:pad + w] = rne_bits(x)
    hh = (torch.arange(P, device='cuda') * stride)[:, None] + torch.arange(r, device='cuda')
    ww = (torch.arange(Q, device='cuda') * stride)[:, None] + torch.arange(s, device='cuda')
    taps = xp[:, :, hh[:, :, None, None], ww[None, None]]                  # [n, c, P, r, Q, s]
    t = torch.zeros(n, P, Q, c, r, _s8(s), device='cuda', dtype=BF16)
    t[..., :s] = taps.permute(0, 2, 4, 1, 3, 5)
    out = torch.zeros(n * P * Q, kpad, device='cuda', dtype=BF16)
    out[:, :c * r * _s8(s)] = t.view(n * P * Q, -1)
    return out


def _prep_ref(w, kpad, order, kp, cp):
    k, c, r, s = w.shape
    wb = rne_bits(w)
    out = torch.zeros(kp, kpad, device='cuda', dtype=BF16)
    if order == ops.ORDER_RSC:
        t = torch.zeros(k, r, s, cp, device='cuda', dtype=BF16)
        t[..., :c] = wb.permute(0, 2, 3, 1)
    else:
        t = torch.zeros(k, c, r, _s8(s), device='cuda', dtype=BF16)
        t[..., :s] = wb
    out[:k, :t[0].numel()] = t.view(k, -1)
    return out


def _cols(c, r, s, order, cp):
    """Column of weight (c, r, s) in the operand layout, int64 [c, r, s]."""
    cc, rr, ss = torch.meshgrid(*(torch.arange(v, device='cuda') for v in (c, r, s)), indexing='ij')
    return (rr * s + ss) * cp + cc if order == ops.ORDER_RSC else (cc * r + rr) * _s8(s) + ss


def _seq_sum(start, terms):
    """start (fp32 or None = +0.0) + terms[0] + terms[1] + ..., one fp32 rounding per add, in that order."""
    s = torch.zeros_like(terms[0]) if start is None else start.clone()
    for t in terms:
        s = fl32_add(s, t)
    return s


def _split_allowance(ref, s, splits):
    """GEMM accumulation allowance of `splits` split-K partials (each within 2^-16 S_j + 2^-22 |ref_j| <= (2^-16 +
    2^-22) S_j), then one fp32 rounding per finish add of a running sum bounded by S."""
    a = acc_allowance(ref, s) + 2.0 ** -22 * s
    for _ in range(splits):
        a = rnd(s, a)
    return a


def _nchw(t, n, h, w):
    return t.view(n, h, w, -1).permute(0, 3, 1, 2)


# ------------------------------------------------------------------ cases
STEM = [  # name, n, c, h, w, r (= s), stride, pad, kpad (0: ops.stem_kpad)
    ('resnet 7x7/2 224', 2, 3, 224, 224, 7, 2, 3, 0),
    ('detr 7x7/2 201x157', 1, 3, 201, 157, 7, 2, 3, 0),
    ('cifar 3x3/1 32', 8, 3, 32, 32, 3, 1, 1, 0),
    ('cifar 3x3/1 64', 4, 3, 64, 64, 3, 1, 1, 0),
    ('van 7x7/4 pad 3', 2, 3, 224, 224, 7, 4, 3, 0),
    ('convformer 7x7/4 pad 2', 2, 3, 224, 224, 7, 4, 2, 0),
    ('vit 16/16 224', 2, 3, 224, 224, 16, 16, 0, 0),
    ('sam 16/16 1024', 1, 3, 1024, 1024, 16, 16, 0, 0),
    ('1 channel', 2, 1, 37, 45, 7, 2, 3, 0),
    ('4 channels', 2, 4, 50, 61, 5, 3, 2, 0),
    ('kpad above stem_kpad', 2, 3, 60, 52, 7, 2, 3, ops.stem_kpad(3, 7, 7) + 72),
    ('56/56 patches', 2, 3, 224, 168, 56, 56, 0, 0),
    ('64/64 patches at 48 KiB', 1, 3, 128, 192, 64, 64, 0, 0),
]
PREP = [  # name, k, c, r, s, order, kp, cp, kpad above the minimum
    ('darknet 32 filters -> 64', 32, 64, 3, 3, 0, 64, 64, 0),
    ('32 channels -> 64', 64, 32, 3, 3, 0, 64, 64, 0),
    ('10-class 1x1 head', 10, 1024, 1, 1, 0, 64, 1024, 0),
    ('unpadded 3x3', 256, 128, 3, 3, 0, 0, 0, 0),
    ('unpadded 1x1', 512, 256, 1, 1, 0, 0, 0, 0),
    ('padded k and c, kpad above', 35, 45, 3, 3, 0, 64, 64, 64),
    ('grid wrap 3x3', 512, 512, 3, 3, 0, 0, 0, 0),
    ('resnet stem', 64, 3, 7, 7, 1, 0, 0, 0),
    ('darknet stem 32 -> 64', 32, 3, 3, 3, 1, 64, 0, 0),
    ('vit-l patch', 1024, 3, 16, 16, 1, 0, 0, 0),
    ('stem kpad above', 64, 3, 7, 7, 1, 0, 0, 72),
]
FINISH = [  # name, k, c, r, s, order, kp, cp, kpad above the minimum, transposed, splits
    ('rsc padded k and c', 32, 48, 3, 3, 0, 64, 64, 0, 0, 7),
    ('rsc padded k and c dW^T', 32, 48, 3, 3, 0, 64, 64, 0, 1, 2),
    ('rsc 10-class 1x1 dW^T', 10, 256, 1, 1, 0, 64, 0, 0, 1, 1),
    ('rsc unpadded 3x3', 128, 64, 3, 3, 0, 0, 0, 0, 0, 64),
    ('rsc kpad above', 64, 64, 3, 3, 0, 0, 0, 64, 0, 2),
    ('crs resnet stem dW^T', 64, 3, 7, 7, 1, 0, 0, 0, 1, 64),
    ('crs darknet stem 32 -> 64 dW^T', 32, 3, 3, 3, 1, 64, 0, 0, 1, 7),
    ('crs vit patch', 96, 3, 16, 16, 1, 0, 0, 0, 0, 2),
    ('crs van stem kpad above', 64, 3, 7, 7, 1, 0, 0, 64, 0, 7),
    ('rsc grid wrap', 512, 256, 3, 3, 0, 0, 0, 0, 0, 2),
]
REDUCE = [  # name, n, splits
    ('conv weight', 64 * 1152, 7),
    ('64 splits', 4096, 64),
    ('grid wrap', 4 * 600000, 3),
    ('one split', 4100, 1),
    ('n % 4 = 1', 3001, 2),
    ('n % 4 = 3', 1023, 7),
]
UPSAMPLE = [(3, 7, 9, 8), (2, 15, 15, 64), (2, 25, 19, 24), (2, 260, 260, 64)]   # N, H, W, C


def _kpad(order, c, r, s, cp, extra):
    return (r * s * (cp or c) if order == ops.ORDER_RSC else ops.stem_kpad(c, r, s)) + extra


def test_cases_cover_every_tile_and_wrap_cpu():
    """The stem cases reach 32, 8 and 1 pixels per block, Q % T != 0 and the 48 KiB patch; the prep, finish, reduce,
    cast, add and scatter cases each have one whose grid-stride loop wraps."""
    tiles = {}
    for name, n, c, h, w, r, stride, pad, kpad in STEM:
        t = _stem_tile(c, r, r, stride)
        tiles.setdefault(t, []).append(name)
        assert c * r * ((t - 1) * stride + r) * 4 <= 48 * 1024, name
        assert not kpad or (kpad % 8 == 0 and kpad > ops.stem_kpad(c, r, r)), name
    assert {32, 8, 1} <= set(tiles), tiles
    assert any(ops.conv_out_size(w, pad, r, stride) % _stem_tile(c, r, r, stride)
               for _, n, c, h, w, r, stride, pad, _ in STEM)
    assert any(c * r * r * 4 == 48 * 1024 for _, n, c, h, w, r, stride, pad, _ in STEM if stride == r)
    assert max((kp or k) * _kpad(o, c, r, s, cp, e) for _, k, c, r, s, o, kp, cp, e in PREP) > CAP
    assert max(k * c * r * s for _, k, c, r, s, *_ in FINISH) > CAP
    assert max(n // 4 for _, n, _ in REDUCE) > CAP
    assert max(n * h * w * c // 8 for n, h, w, c in UPSAMPLE) > CAP
    assert {s for *_, s in FINISH} >= {1, 2, 7, 64} and {s for *_, s in REDUCE} >= {1, 2, 7, 64}


# ------------------------------------------------------------------ stem im2col
@gpu
@pytest.mark.parametrize('case', STEM, ids=[s[0] for s in STEM])
def test_stem_im2col_is_exact(case):
    name, n, c, h, w, r, stride, pad, kpad = case
    kpad = kpad or ops.stem_kpad(c, r, r)
    x = _sprinkle(_wide(n, c, h, w, seed=100), seed=101)
    P, Q = ops.conv_out_size(h, pad, r, stride), ops.conv_out_size(w, pad, r, stride)

    def run():
        cols = nan(n * P * Q, kpad, dtype=BF16)
        call('saicv_stem_im2col', x, cols, n, c, h, w, r, r, stride, pad, kpad)
        return cols

    cols = run()
    exact('stem_im2col', f'stem_im2col {name} (T {_stem_tile(c, r, r, stride)}, kpad {kpad})', cols,
          _stem_ref(x, r, r, stride, pad, kpad))
    same(f'stem_im2col {name} on a second launch', run(), cols)


# ------------------------------------------------------------------ weight operand copy
@gpu
@pytest.mark.parametrize('case', PREP, ids=[p[0] for p in PREP])
def test_prep_conv_weight_is_exact(case):
    name, k, c, r, s, order, kp, cp, extra = case
    kp_, cp_ = kp or k, cp or c
    kpad = _kpad(order, c, r, s, cp_, extra)
    w = _sprinkle(_wide(k, c, r, s, seed=200), seed=201)
    out = nan(kp_, kpad, dtype=BF16)
    call('saicv_prep_conv_weight', w, out, k, c, r, s, kpad, order, kp, cp)
    exact('prep_conv_weight', f'prep_conv_weight {name} ({k}x{c}x{r}x{s} -> {kp_}x{kpad}, order {order})', out,
          _prep_ref(w, kpad, order, kp_, cp_))


# ------------------------------------------------------------------ weight-gradient finish
@gpu
@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('case', FINISH, ids=[f[0] for f in FINISH])
def test_finish_conv_wgrad_is_sequential_and_reads_only_the_map(case, accumulate):
    """Every partial position outside the map (padded filters and channels, S8 and tail columns) is NaN."""
    name, k, c, r, s, order, kp, cp, extra, tr, splits = case
    kp_, cp_ = kp or k, cp or c
    kpad = _kpad(order, c, r, s, cp_, extra)
    vals = randn(splits, k, c * r * s, seed=300) * torch.exp2(torch.randint(-6, 6, (splits, 1, 1), device='cuda',
                                                                             generator=gen(301)).float())
    zeros = rand(splits, k, c * r * s, seed=302) < 0.05
    vals = torch.where(zeros, torch.where(rand(splits, k, c * r * s, seed=303) < 0.5, 0.0, -0.0), vals)
    vals[:, :, :3] = _f32_bits([0x80000000, 0x00000001, 0x807FFFFF])           # -0.0 and subnormals in every split
    col = _cols(c, r, s, order, cp_).flatten()
    kk = torch.arange(k, device='cuda')
    if tr:
        part = nan(splits, kpad, kp_)
        part[:, col[:, None], kk[None, :]] = vals.transpose(1, 2)
    else:
        part = nan(splits, kp_, kpad)
        part[:, kk[:, None], col[None, :]] = vals
    g0 = randn(k, c * r * s, seed=304)
    g0[:, :2] = _f32_bits([0x80000000, 0x00000000])
    grad = g0.clone() if accumulate else nan(k, c * r * s)
    call('saicv_finish_conv_wgrad', part, grad, splits, k, c, r, s, kpad, accumulate, order, kp, cp, tr)
    what = f'finish_conv_wgrad {name} splits {splits}{" accumulate" if accumulate else ""}'
    v = vals.double().sum(0) + (g0.double() if accumulate else 0)
    mag = vals.double().abs().sum(0) + (g0.double().abs() if accumulate else 0)
    check('finish_conv_wgrad', what, grad, v, (splits + 1) * U * mag)
    exact('finish_conv_wgrad order', f'{what}: ascending split order', grad,
          _seq_sum(g0 if accumulate else None, list(vals)))


# ------------------------------------------------------------------ split-K reduction
def _reduce(partial, out0, accumulate, offset_partial=False, offset_out=False):
    """saicv_reduce_partials on copies of partial / out0, placed 1 element past a 16-byte boundary when asked."""
    splits, n = partial.shape

    def place(t, off):
        if not off:
            return t.clone()
        buf = torch.empty(t.numel() + 1, device='cuda', dtype=t.dtype)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        return v

    p, o = place(partial, offset_partial), place(out0, offset_out)
    call('saicv_reduce_partials', p, o, splits, n, accumulate)
    return o


@gpu
@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('case', REDUCE, ids=[r[0] for r in REDUCE])
def test_reduce_partials_is_sequential_on_both_paths(case, accumulate):
    name, n, splits = case
    partial = randn(splits, n, seed=400) * torch.exp2(torch.randint(-8, 8, (splits, 1), device='cuda',
                                                                    generator=gen(401)).float())
    partial[:, :4] = _f32_bits([0x80000000, 0x00000001, 0x807FFFFF, 0x00000000])
    out0 = randn(n, seed=402) if accumulate else nan(n)
    if accumulate:
        out0[:2] = _f32_bits([0x80000000, 0x00000000])
    want = _seq_sum(out0 if accumulate else None, list(partial))
    what = f'reduce_partials {name} splits {splits}{" accumulate" if accumulate else ""}'
    paths = {'float4' if n % 4 == 0 else 'scalar': (False, False), 'scalar, partial offset': (True, False),
             'scalar, out offset': (False, True)}
    for path, (op, oo) in paths.items():
        exact('reduce_partials', f'{what} ({path})', _reduce(partial, out0, accumulate, op, oo), want)


# ------------------------------------------------------------------ fp32 -> bf16 cast
def _every_upper_half():
    """Every fp32 upper half x low halves {0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF}: 393216 values."""
    hi = torch.arange(1 << 16, device='cuda', dtype=torch.int64)
    lo = torch.tensor([0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF], device='cuda', dtype=torch.int64)
    u = ((hi[:, None] << 16) | lo[None, :]).flatten()
    return torch.where(u >= 1 << 31, u - (1 << 32), u).to(torch.int32).view(F32)


def _cast(x, path):
    n = x.numel()
    if path == 'vector':
        src, dst = x, nan(n, dtype=BF16)
    elif path == 'scalar n % 8':
        n -= 3
        src, dst = x[:n].clone(), nan(n, dtype=BF16)
    elif path == 'scalar src offset':
        buf = torch.empty(n + 1, device='cuda')
        src, dst = buf[1:], nan(n, dtype=BF16)
        src.copy_(x)
    else:
        src, dst = x, nan(n + 1, dtype=BF16)[1:]
    call('saicv_cast_bf16', src, dst, n)
    return src, dst


CAST_PATHS = ['vector', 'scalar n % 8', 'scalar src offset', 'scalar dst offset']


@gpu
@pytest.mark.parametrize('path', CAST_PATHS)
def test_cast_bf16_rounds_every_upper_half(path):
    src, dst = _cast(_every_upper_half(), path)
    _exact_or_nan('cast_bf16', f'cast_bf16 every upper half ({path})', dst, src)


@gpu
@pytest.mark.parametrize('path', CAST_PATHS)
def test_cast_bf16_streams(path):
    """4.8 M values: both kernels' grid-stride loops wrap."""
    src, dst = _cast(_sprinkle(_wide(8 * 600000, seed=500), seed=501), path)
    _exact_or_nan('cast_bf16', f'cast_bf16 n {src.numel()} ({path})', dst, src)


# ------------------------------------------------------------------ bf16 adds
def _add_operands(n, seed):
    """bf16 pairs: wide random values, exact cancellations, exponent gaps of 17..30, -0 + -0, and the specials."""
    a = _wide(n, seed=seed).to(BF16)          # the cast is only an input generator here
    b = _wide(n, seed=seed + 1).to(BF16)
    pick = torch.randint(0, 8, (n,), device='cuda', generator=gen(seed + 2))
    gap = torch.exp2(-torch.randint(17, 31, (n,), device='cuda', generator=gen(seed + 3)).float())
    sign = torch.where(rand(n, seed=seed + 4) < 0.5, -1.0, 1.0)
    b = torch.where(pick == 0, -a, b)
    b = torch.where(pick == 1, (a.float() * gap * sign * (1 + rand(n, seed=seed + 5))).to(BF16), b)
    spec = _bf16_bits(BF16_SPECIALS)
    r = lambda s: spec[torch.randint(0, spec.numel(), (n,), device='cuda', generator=gen(seed + s))]  # noqa: E731
    a = torch.where(pick == 2, r(6), a)
    b = torch.where((pick == 2) | (pick == 3), r(7), b)
    a[:2], b[:2] = _bf16_bits([0x8000, 0x8000]), _bf16_bits([0x8000, 0x0000])
    return a.contiguous(), b.contiguous()


@gpu
@pytest.mark.parametrize('n', [8 * 37, 8 * 600000])
def test_add_bf16_is_fp32_sum_rounded_once(n):
    a, b = _add_operands(n, seed=600)
    out = a.clone()
    call('saicv_add_bf16', out, b, n)
    _exact_or_nan('add_bf16', f'add_bf16 n {n}', out, fl32_add(a, b))
    cancel = (b == -a) & (a != 0) & torch.isfinite(a.float())
    assert cancel.sum() > n // 16 and (out[cancel].view(torch.int16) == 0).all(), 'add_bf16: a + (-a) is not +0.0'


# ------------------------------------------------------------------ stride-2 scatters
@gpu
@pytest.mark.parametrize('n,h,w,c', UPSAMPLE)
def test_zero_upsample2_is_exact(n, h, w, c):
    P, Q = (h + 1) // 2, (w + 1) // 2
    dy = rne_bits(_sprinkle(_wide(n, P, Q, c, seed=700), seed=701))
    dy.view(-1)[:4] = _bf16_bits([0x7FC1, 0xFFA5, 0x8000, 0x0001])        # NaN payloads are copied bit for bit
    u = nan(n, h, w, c, dtype=BF16)
    call('saicv_zero_upsample2', dy, u, n, P, Q, h, w, c)
    want = torch.zeros(n, h, w, c, device='cuda', dtype=BF16)
    want[:, ::2, ::2] = dy
    exact('zero_upsample2', f'zero_upsample2 {n}x{P}x{Q}x{c} -> {h}x{w}', u, want)


@gpu
@pytest.mark.parametrize('n,h,w,c', UPSAMPLE)
def test_add_strided2_touches_only_even_pixels(n, h, w, c):
    P, Q = (h + 1) // 2, (w + 1) // 2
    a, b = _add_operands(n * P * Q * c, seed=800)
    dx = nan(n, h, w, c, dtype=BF16)
    dx[:, ::2, ::2] = a.view(n, P, Q, c)
    want = dx.clone()
    dd = b.view(n, P, Q, c)
    call('saicv_add_strided2', dx, dd, n, P, Q, h, w, c)
    what = f'add_strided2 {n}x{P}x{Q}x{c} -> {h}x{w}'
    _exact_or_nan('add_strided2', what, dx[:, ::2, ::2], fl32_add(a, b).view(n, P, Q, c))
    want[:, ::2, ::2] = dx[:, ::2, ::2]
    same(f'{what}: the odd rows and columns', dx, want)


# ------------------------------------------------------------------ compositions
STEM_COMP = [  # name, n, h, k, r, stride, pad
    ('resnet 7x7/2', 2, 224, 64, 7, 2, 3),
    ('vit 16/16', 2, 224, 768, 16, 16, 0),
]


@gpu
@pytest.mark.parametrize('case', STEM_COMP, ids=[s[0] for s in STEM_COMP])
def test_stem_layouts_agree_through_the_gemm(case):
    """stem_im2col + prep_conv_weight(order 1) + linear_fwd = conv2d; linear_wgrad + finish_conv_wgrad(order 1) =
    conv2d_weight, in the orientation the conv runtime picks (wgrad_transposed(kp, kpad))."""
    name, n, h, k, r, stride, pad = case
    c, kp, kpad = 3, (k + 63) // 64 * 64, ops.stem_kpad(3, r, r)
    x = randn(n, c, h, h, seed=900)
    wt = randn(k, c, r, r, scale=(c * r * r) ** -0.5, seed=901)
    P = ops.conv_out_size(h, pad, r, stride)
    M = n * P * P
    cols = ops.stem_im2col(x, r, r, stride, pad, kpad)
    wb = nan(kp, kpad, dtype=BF16)
    ops.prep_conv_weight(wt, wb, kpad, order=ops.ORDER_CRS, kp=kp)
    y = ops.linear_fwd(cols, wb)
    xr, wr = rne_bits(x).double(), rne_bits(wt).double()
    ref = F.conv2d(xr, wr, stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(M, k)
    s = F.conv2d(xr.abs(), wr.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(M, k)
    check('stem forward', f'stem {name} forward', y[:, :k], ref, acc_allowance(ref, s), s)
    assert (y[:, k:] == 0).all(), f'stem {name}: padded filters gave non-zero outputs'

    dy = randn(M, kp, scale=M ** -0.5, seed=902).to(BF16)
    tr = ops.wgrad_transposed(kp, kpad)
    part = ops.linear_wgrad(dy, cols, transposed=tr)
    grad = nan(k, c, r, r)
    call('saicv_finish_conv_wgrad', part, grad, part.shape[0], k, c, r, r, kpad, 0, ops.ORDER_CRS, kp, 0, int(tr))
    dyd = _nchw(dy.double(), n, P, P)[:, :k]
    ref = conv2d_weight(xr, grad.shape, dyd, stride=stride, padding=pad)
    s = conv2d_weight(xr.abs(), grad.shape, dyd.abs(), stride=stride, padding=pad)
    check('stem weight gradient', f'stem {name} weight gradient{" (dW^T)" if tr else ""}, {part.shape[0]} splits',
          grad, ref, _split_allowance(ref, s, part.shape[0]), s)


PADDED = [  # n, h, c, k, r, stride, pad, transposed
    (4, 28, 32, 32, 3, 1, 1, True),      # DarkNet-like: 32 filters and channels padded to 64
    (4, 20, 100, 200, 3, 1, 1, False),
]


@gpu
@pytest.mark.parametrize('n,h,c,k,r,stride,pad,transposed', PADDED)
def test_padded_conv_weight_gradient_agrees(n, h, c, k, r, stride, pad, transposed):
    cp, kp = (c + 63) // 64 * 64, (k + 63) // 64 * 64
    ncols = r * r * cp
    assert ops.wgrad_transposed(kp, ncols) == transposed
    x = torch.zeros(n, h, h, cp, device='cuda', dtype=BF16)
    x[..., :c] = randn(n, h, h, c, seed=1000).to(BF16)
    P = ops.conv_out_size(h, pad, r, stride)
    dy = randn(n, P, P, kp, scale=(n * P * P) ** -0.5, seed=1001).to(BF16)
    part = ops.conv_wgrad(dy, x, ops.make_conv_shape(n, h, h, cp, kp, r, r, stride, pad))
    grad = nan(k, c, r, r)
    call('saicv_finish_conv_wgrad', part, grad, part.shape[0], k, c, r, r, ncols, 0, ops.ORDER_RSC, kp, cp,
         int(transposed))
    xd, dyd = x.double().permute(0, 3, 1, 2)[:, :c], dy.double().permute(0, 3, 1, 2)[:, :k]
    ref = conv2d_weight(xd, grad.shape, dyd, stride=stride, padding=pad)
    s = conv2d_weight(xd.abs(), grad.shape, dyd.abs(), stride=stride, padding=pad)
    check('padded conv weight gradient',
          f'conv {k}->{kp} filters {c}->{cp} channels{" (dW^T)" if transposed else ""}, {part.shape[0]} splits',
          grad, ref, _split_allowance(ref, s, part.shape[0]), s)


# ------------------------------------------------------------------ refusals
def _refusals(f):
    """(entry, args without the stream, message fragment); f: an fp32 buffer large enough for every shape here, so no
    call could read or write outside it even if it launched."""
    return [
        ('saicv_stem_im2col', (f, f, 1, 3, 16, 16, 7, 7, 2, 3, 172), 'must be a multiple of 8'),
        ('saicv_stem_im2col', (f, f, 1, 3, 16, 16, 7, 7, 2, 3, 160), 'must be a multiple of 8 >= c*r*roundup(s, 8) = 168'),
        ('saicv_stem_im2col', (f, f, 1, 4, 64, 64, 64, 64, 64, 0, 4 * 64 * 64), 'does not fit in shared memory'),
        ('saicv_prep_conv_weight', (f, f, 4, 8, 3, 3, 76, 0, 0, 0), 'bad padding'),
        ('saicv_prep_conv_weight', (f, f, 4, 8, 3, 3, 64, 0, 0, 0), 'bad padding'),
        ('saicv_prep_conv_weight', (f, f, 4, 8, 3, 3, 72, 0, 0, 16), 'bad padding'),
        ('saicv_prep_conv_weight', (f, f, 4, 3, 7, 7, 152, 1, 0, 0), 'bad padding'),
        ('saicv_prep_conv_weight', (f, f, 4, 8, 3, 3, 72, 0, 2, 0), 'bad padding'),
        ('saicv_prep_conv_weight', (f, f, 4, 8, 3, 3, 72, 0, 0, 4), 'bad padding'),
        ('saicv_add_bf16', (f, f, 12), 'n % 8'),
        ('saicv_zero_upsample2', (f, f, 1, 2, 2, 4, 4, 12), 'C % 8'),
        ('saicv_add_strided2', (f, f, 1, 2, 2, 4, 4, 12), 'C % 8'),
    ]


@gpu
def test_refusals_launch_nothing():
    """kpad not a multiple of 8 or below the column map (stem_im2col; prep_conv_weight in either order), a stem patch
    that does not fit in shared memory, kp < k, cp < c, n % 8 (add_bf16), C % 8 (the scatters): an error, no launch."""
    f = torch.zeros(1 << 20, device='cuda')
    for name, args, msg in _refusals(f):
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            call(name, *args)
        assert _lib.launch_count() == n0, f'{name}{args[2:]}: launched before refusing'
    torch.cuda.synchronize()
