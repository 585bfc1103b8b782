"""Conformance of the normalisation, column-sum and pooling kernels against a float64 reference, and their bit-identity
invariants.

Reference.  Every check computes the exact result in float64 on the GPU from the same bf16 / fp32 inputs the kernel
read.  A kernel that consumes the stored output of an earlier kernel (bn_apply reads scale_shift, the backward kernels
read the saved mean / rstd and the folded sums) is checked against the exact operation on those stored values, and
the earlier kernel is checked on its own; so each allowance belongs to one kernel.

Allowances are derived from the operation, never fitted to measured errors (u = 2^-24, one fp32 rounding):
  * fp32 sums.  A sum of n terms reduced in a tree of depth d is within (d + 1) u sum|terms| of the exact sum.  d is
    taken from a Python mirror of each launch's geometry: slab_geom / partial_rows of capi_elementwise.cu, slab of
    capi_van.cu, grid_1d of the LayerNorm backwards.  For a slab reduction d = the per-thread chain (rows per block /
    ty_count) + log2(ty_count) (the tree fold) + ceil(nblk / 32) + 32 (the fold of the partial rows); the generic
    BatchNorm folds its ty_count rows and, in the backward, its partial rows sequentially.  Sequential kernels (fp32
    colsum, avgpool) have d = the number of terms.  A term that is itself a product of rounded factors adds its own
    rounding count times u |term|.
  * Derived quantities carry the allowance through every operation: one fp32 rounding per operation (1 / n counts
    as one), rsqrtf at 2 ulp (2^-22 relative), evaluated as an interval: rstd must lie in
    [rsqrt(var + a_var + eps), rsqrt(max(var - a_var, 0) + eps)] widened by 2^-22.  The BatchNorm variance is one-pass,
    E[x^2] - mean^2 in fp32, so its allowance is stated in sum(x^2) / n = var + mean^2: a_var ~ (d + 4) u (var +
    mean^2), and the relative rstd allowance grows as (d + 4) u (1 + (mean / std)^2) / 2.  At |mean| / std = 64 and
    d ~ 60 the variance allowance is about 1.6e-2 of var; at 512 (fp32 input) it exceeds var itself, so rstd is then
    bounded only through eps: the one-pass formula guarantees nothing there.  The offset cases print the measured
    error next to torch's fp32 batch_norm.
  * bn_bwd_apply adds A g + B y + K with A = gamma rstd, B = -A rstd k3, K = -A k2 + A rstd k3 mean; its allowance is
    10 u (|A g| + |B y| + |A k2| + |A rstd k3 mean|) plus |A| times the allowance of the masked gradient: when
    |mean| >> std the two large terms B y and K cancel, and the allowance grows with them.
  * ReLU, the 0/1 masks and LeakyReLU are 1-Lipschitz (LeakyReLU's 0.1f and its product add 2 u |out|).  SiLU uses
    |silu'| <= 1.1 and |silu''| <= 0.5 plus SILU_ABS for the fast-math __expf / __fdividef, which is checked on every
    finite bf16 input by test_silu_fast_math_on_every_bf16_input.  A recomputed ReLU mask whose pre-activation lies
    within its rounding allowance of 0 may go either way, so that element's gradient allowance is |g|.
  * Running statistics follow torch's documented update: r = (1 - m) r + m x with the unbiased variance
    var * rows / (rows - 1).
  * Max-pool: the forward value and argmax are bit-exact against a float64 reference that applies torch's rule (the
    first maximum in (r, s) scan order wins; -inf padding never wins, a zero-padded tap carries code 255).  The
    backward adds at most ceil(k / stride)^2 bf16 gradients, so it gets that many roundings.

Invariants (raw bits): two consecutive launches of every kernel give identical outputs, and bn_finalize with
partial_rows = 0 equals the call given the partial-row count of the Python mirror of slab_geom (a disagreement
between partial_rows() and the stats launch would drop or double a block).  Partial workspaces and outputs are
filled with NaN before each launch, so an unwritten element or a folded stale row fails.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conformance import (NAN, PARTIAL_ROWS, U, check, every_bf16, gen, nan, next_pow2, quantum_bf16, rand, randn, rnd,
                         rne_bf16, same, van_slab)
from conformance import report  # noqa: F401  (autouse: this module's allowance report)

from simpleaicv_pytorch_training_examples_b200 import ops

pytestmark = pytest.mark.gpu

RSQRT = 2.0 ** -22      # rsqrtf: 2 ulp, relative
SILU_ABS = 4e-6         # |fast-math silu - silu| and |fast-math silu' - silu'| beyond their final roundings
LEAKY = 0.1


def _same_all(what, a, b):
    for k in a:
        if a[k] is not None:
            same(f'{what}: {k} on a second launch', a[k], b[k])


# ------------------------------------------------------------------ launch geometry mirrors
def _slab(rows, c, unroll, max_blocks=PARTIAL_ROWS):
    """capi_elementwise.cu slab_geom: (ty_count, rows_per_block, blocks)."""
    tx = min(next_pow2(c // 8), 256)
    ty = 256 // tx
    b = max(1, min(-(-rows // (ty * unroll)), max_blocks))
    q = ty * unroll
    rpb = -(-(-(-rows // b)) // q) * q
    return ty, rpb, -(-rows // rpb)


def _slab_depth(rows, c, unroll, accumulate=False):
    """Depth of a slab column reduction (colreduce_kernel / colreduce2_kernel) folded by fold_partials / bn_finalize."""
    ty, rpb, nblk = _slab(rows, c, unroll)
    return -(-rpb // ty) + int(math.log2(ty)) + -(-nblk // 32) + 32 + int(accumulate)


def _ln_bwd_depth(rows, accumulate=False):
    """ln_bwd_kernel / postln_bwd_kernel (grid_1d(rows, 64, 264) blocks of 8 warps) + fold_partials_kernel."""
    grid = max(1, min(-(-rows // 64), 264))
    return -(-rows // (grid * 8)) + 8 + -(-grid // 32) + 32 + int(accumulate)


# ------------------------------------------------------------------ activations
def _act64(v, act):
    if act == 1:
        return v.clamp_min(0)
    if act == 2:
        return torch.where(v > 0, v, LEAKY * v)
    if act == 3:
        return v * torch.sigmoid(v)
    return v


def _act_allow(v, a, act):
    """Allowance of act_apply on a value within a of v (including the rounding of act_apply's own product)."""
    if act == 2:
        return a + 2 * U * _act64(v, act).abs()
    if act == 3:
        return 1.1 * a + SILU_ABS + 2 * U * _act64(v, act).abs()
    return a


def _silu_grad64(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s)), SILU_ABS + 4 * U * s * (1 + z.abs())


def _unpack_bits(bits, c):
    b = bits.view(torch.uint8).long()   # little-endian: byte k of a word holds channels 8k .. 8k+7 of it
    return ((b.unsqueeze(-1) >> torch.arange(8, device=b.device)) & 1).reshape(b.shape[0], c).double()


def _grad_factor(act, src, y, out, bits, ss):
    """(f, a_f): act'(.) as the backward kernels form it from mask source src, and its allowance."""
    if act == 0:
        return 1.0, 0.0
    if src == 'bits':
        return _unpack_bits(bits, y.shape[1]), 0.0
    lo = 0.0 if act == 1 else LEAKY
    if src == 'out':
        return (out.double() > 0).double() * (1 - lo) + lo, 0.0
    t = y.double() * ss[0].double()
    z = t + ss[1].double()
    a_z = 2 * U * (t.abs() + ss[1].double().abs())
    if act == 3:
        f, a = _silu_grad64(z)
        return f, 0.5 * a_z + a
    return (z > 0).double() * (1 - lo) + lo, (z.abs() <= a_z).double() * (1 - lo)


# ------------------------------------------------------------------ BatchNorm references
def _stats_allow(x64, depth):
    """Exact mean / biased variance of x64 [rows, C] and the allowances of the one-pass fp32 mean and variance."""
    n = x64.shape[0]
    mean = x64.sum(0) / n
    var = ((x64 - mean) ** 2).sum(0) / n
    ex2 = (x64 * x64).sum(0) / n
    e0 = (depth + 1) * U * x64.abs().sum(0) / n
    e1 = (depth + 1) * U * ex2
    a_m = e0 + 3 * U * (mean.abs() + e0)
    a_ex2 = e1 + 3 * U * (ex2 + e1)
    a_msq = 2 * mean.abs() * a_m + a_m * a_m + 3 * U * (mean.abs() + a_m) ** 2
    a_v = a_ex2 + a_msq + 2 * U * (var + a_ex2 + a_msq)
    return mean, var, a_m, a_v


def _rstd_interval(var, a_v, eps):
    """Exact rstd and the half-width of the interval the rsqrtf of an fp32 variance within a_v of var may take."""
    e = torch.tensor(eps, dtype=torch.float32).double().item()
    r = (var + e).rsqrt()
    t_lo = ((var - a_v).clamp_min(0) + e) * (1 - 2 * U)      # + eps rounds once; the kernel clamps var at 0
    t_hi = (var + a_v + e) * (1 + 2 * U)
    return r, torch.maximum(t_lo.rsqrt() * (1 + RSQRT) - r, r - t_hi.rsqrt() * (1 - RSQRT))


def _check_finalize(fam, what, x, gamma, beta, eps, mom, rm0, rv0, o, depth):
    """bn_finalize outputs o = {ss, saved, rm, rv} against the exact statistics of x."""
    n = x.shape[0]
    mean, var, a_m, a_v = _stats_allow(x.double(), depth)
    r, a_r = _rstd_interval(var, a_v, eps)
    g, b = gamma.double(), beta.double()
    check(fam, f'{what} mean', o['saved'][0], mean, a_m)
    check(fam, f'{what} rstd', o['saved'][1], r, a_r)
    sc = g * r
    a_sc = g.abs() * a_r + U * g.abs() * (r + a_r)
    sh = b - mean * sc
    # mean * scale and beta - that: two roundings of values within (a_m, a_sc) of the exact factors
    a_sh = mean.abs() * a_sc + (sc.abs() + a_sc) * a_m + 2 * U * ((mean.abs() + a_m) * (sc.abs() + a_sc) + b.abs())
    check(fam, f'{what} scale', o['ss'][0], sc, a_sc)
    check(fam, f'{what} shift', o['ss'][1], sh, a_sh)
    if rm0 is not None:
        # (1 - m) r + m x in fp32: 1 - m, two products and the sum round (4u), and 0.1f differs from 0.1 by 1.5e-8
        # relative (under u); the unbiased factor rows / (rows - 1) and its product add two more
        rm = (1 - mom) * rm0.double() + mom * mean
        a_rm = mom * a_m + 5 * U * ((1 - mom) * rm0.double().abs() + mom * (mean.abs() + a_m))
        unb = n / (n - 1) if n > 1 else 1.0
        rv = (1 - mom) * rv0.double() + mom * unb * var
        a_rv = mom * unb * a_v + 7 * U * ((1 - mom) * rv0.double().abs() + mom * unb * (var + a_v))
        check(fam, f'{what} running_mean', o['rm'], rm, a_rm)
        check(fam, f'{what} running_var', o['rv'], rv, a_rv)
    return r, a_r


def _bn_forward(y, gamma, beta, eps, mom, rm0, rv0, partial_rows=0):
    c = y.shape[1]
    ws = ops.partial_ws(y.device, 2 * c)
    ws.fill_(NAN)
    ops.bn_stats(y, ws)
    o = {'ss': nan(2, c), 'saved': nan(2, c),
         'rm': rm0.clone() if rm0 is not None else None, 'rv': rv0.clone() if rv0 is not None else None}
    ops.bn_finalize(ws, gamma, beta, o['rm'], o['rv'], o['ss'], o['saved'], y.shape[0], eps, mom, partial_rows=partial_rows)
    return o


def _apply_ref(y, ss, act, res, rss):
    """Exact bn_apply output from the stored scale_shift (and the residual's), with its allowance."""
    t = y.double() * ss[0].double()
    v = t + ss[1].double()
    a = 2 * U * (t.abs() + ss[1].double().abs())
    r, a_r = 0.0, 0.0
    if res is not None:
        r = res.double()
        if rss is not None:
            tr = r * rss[0].double()
            r = tr + rss[1].double()
            a_r = 2 * U * (tr.abs() + rss[1].double().abs())
    if act & 8:
        f = _act64(v, act & 7)
        a = _act_allow(v, a, act & 7)
        if res is not None:
            f = f + r
            a = rnd(f, a + a_r)
        return f, a
    if res is not None:
        v = v + r
        a = rnd(v, a + a_r)
    return _act64(v, act), _act_allow(v, a, act)


def _check_bwd(fam, what, dout, y, saved, gamma, f, a_f, o, depth, prev=None):
    """bn_bwd_reduce sums, dgamma / dbeta, dres and dy (o: the kernel outputs) against the exact backward of the
    masked gradient ge = dout * f.  The data gradient is checked from the kernel's own folded sums."""
    n = y.shape[0]
    g = dout.double()
    ge = g * f
    a_ge = g.abs() * a_f + 2 * U * ge.abs()
    mean, rstd = saved[0].double(), saved[1].double()
    y64 = y.double()
    xh = (y64 - mean) * rstd
    t1 = ge * xh
    s0, s1 = ge.sum(0), t1.sum(0)
    a0 = (depth + 1) * U * ge.abs().sum(0) + a_ge.sum(0)
    a1 = (depth + 1) * U * t1.abs().sum(0) + (a_ge * xh.abs() + 3 * U * t1.abs()).sum(0)
    check(fam, f'{what} sum g', o['sums'][0], s0, a0)
    check(fam, f'{what} sum g*xhat', o['sums'][1], s1, a1)
    if prev is None:
        check(fam, f'{what} dbeta', o['dbeta'], s0, a0)
        check(fam, f'{what} dgamma', o['dgamma'], s1, a1)
    else:
        v0, v1 = prev[1].double() + s0, prev[0].double() + s1
        check(fam, f'{what} dbeta (accumulate)', o['dbeta'], v0, rnd(v0, a0))
        check(fam, f'{what} dgamma (accumulate)', o['dgamma'], v1, rnd(v1, a1))
    del t1
    if o.get('dres') is not None:
        check(fam, f'{what} dres', o['dres'], ge, a_ge)
    A = gamma.double() * rstd
    k2, k3 = o['sums'][0].double() / n, o['sums'][1].double() / n
    T1, T2, B = A * k2, A * k3 * rstd * mean, -A * k3 * rstd
    By = B * y64
    v = A * ge + By + (T2 - T1)
    a = A.abs() * a_ge + 10 * U * ((A * ge).abs() + By.abs() + T1.abs() + T2.abs())
    check(fam, f'{what} dy', o['dy'], v, a)


def _bn_backward(dout, y, saved, gamma, ss, act, src, out, bits, want_dres, accumulate=False, prev=None):
    c = y.shape[1]
    o = {'sums': nan(2, c), 'dy': torch.full_like(y, NAN), 'dres': torch.full_like(y, NAN) if want_dres else None,
         'dgamma': prev[0].clone() if accumulate else nan(c), 'dbeta': prev[1].clone() if accumulate else nan(c)}
    mo = out if src == 'out' else None
    mb = bits if src == 'bits' else None
    ms = ss if src == 'recompute' else None
    ops.bn_bwd_reduce(dout, mo, y, saved, o['sums'], act, scale_shift=ms, bits=mb)
    ops.bn_bwd_apply(dout, mo, y, saved, gamma, o['sums'], o['dy'], o['dres'], o['dgamma'], o['dbeta'], act,
                     accumulate=accumulate, scale_shift=ms, bits=mb)
    return o


def _bn_case(rows, c, seed, offset=1.0):
    """y bf16 [rows, c] with per-channel |mean| / std up to `offset`, gamma (either sign), beta, running stats."""
    std = rand(c, seed=seed) * 1.5 + 0.5
    mean = (rand(c, seed=seed + 1) * 2 - 1) * offset * std
    y = (randn(rows, c, seed=seed + 2) * std + mean).to(torch.bfloat16)
    gamma = randn(c, seed=seed + 3) * 0.5 + 1.0
    beta = randn(c, seed=seed + 4) * 0.5
    rm0, rv0 = randn(c, seed=seed + 5) * 0.1, rand(c, seed=seed + 6) + 0.5
    return y, gamma, beta, rm0, rv0


def _run_slab_bn(rows, c, act, res_kind, srcs, seed, accumulate=(False,), what=''):
    """Forward (stats, finalize, apply) and backward (reduce, apply) for each mask source; returns the raw outputs."""
    y, gamma, beta, rm0, rv0 = _bn_case(rows, c, seed)
    res = randn(rows, c, seed=seed + 7).to(torch.bfloat16) if res_kind != 'none' else None
    rss = torch.stack([rand(c, seed=seed + 8) + 0.5, randn(c, seed=seed + 9) * 0.5]) if res_kind == 'bn' else None
    dout = randn(rows, c, seed=seed + 10).to(torch.bfloat16)
    fo = _bn_forward(y, gamma, beta, 1e-5, 0.1, rm0, rv0)
    out = torch.full_like(y, NAN)
    bits = ops.mask_bits_like(y) if 'bits' in srcs else None
    ops.bn_apply(y, fo['ss'], out, act, res=res, res_scale_shift=rss, mask_bits=bits)
    outs = {'fwd': fo, 'out': out, 'bits': bits, 'bwd': {}}
    for src in srcs:
        for acc in accumulate:
            prev = (randn(c, seed=seed + 11), randn(c, seed=seed + 12)) if acc else None
            outs['bwd'][(src, acc)] = (_bn_backward(dout, y, fo['saved'], gamma, fo['ss'], act & 7, src, out, bits,
                                                    want_dres=res_kind == 'plain' and not act & 8,
                                                    accumulate=acc, prev=prev), prev)
    return (y, gamma, beta, rm0, rv0, res, rss, dout), outs


def _check_slab_bn(fam, what, inputs, outs, rows, c, act):
    y, gamma, beta, rm0, rv0, res, rss, dout = inputs
    fo = outs['fwd']
    _check_finalize(fam + ' stats', what, y, gamma, beta, 1e-5, 0.1, rm0, rv0, fo, _slab_depth(rows, c, 8))
    v, a = _apply_ref(y, fo['ss'], act, res, rss)
    check(fam + ' apply', f'{what} out', outs['out'], v, a)
    del v, a
    for (src, acc), (o, prev) in outs['bwd'].items():
        f, a_f = _grad_factor(act & 7, src, y, outs['out'], outs['bits'], fo['ss'])
        _check_bwd(fam + ' backward', f'{what} bwd[{src}{" acc" if acc else ""}]', dout, y, fo['saved'], gamma, f, a_f,
                   o, _slab_depth(rows, c, 4), prev=prev)


def _flatten(outs):
    d = {'ss': outs['fwd']['ss'], 'saved': outs['fwd']['saved'], 'rm': outs['fwd']['rm'], 'rv': outs['fwd']['rv'],
         'out': outs['out'], 'bits': outs['bits']}
    for (src, acc), (o, _) in outs['bwd'].items():
        for k, t in o.items():
            d[f'{k}[{src},{acc}]'] = t
    return d


# ------------------------------------------------------------------ SiLU fast math, on every bf16 input
def test_silu_fast_math_on_every_bf16_input():
    """SiLU forward (bn_apply act 3|8) and its gradient (the recompute mask of bn_bwd_reduce) on every finite bf16
    value, with scale 1 and shift 0 so the activation sees the bf16 value itself.
    Forward: the residual is -rne(silu(y)), so the bf16 output resolves the fp32 silu to about 2^-9 of its error.
    Gradient: one row per launch, so sum g = silu'(y) exactly as the kernel formed it (every other addend is 0)."""
    c = 256
    y = every_bf16(c)
    rows = y.shape[0]
    ss = torch.stack([torch.ones(c, device='cuda'), torch.zeros(c, device='cuda')])
    f64 = _act64(y.double(), 3)
    res = rne_bf16(-f64).to(torch.bfloat16)
    out = torch.full_like(y, NAN)
    ops.bn_apply(y, ss, out, 3 | 8, res=res)
    v, a = _apply_ref(y, ss, 3 | 8, res, None)
    o = out.double()
    err = (((o - v).abs() - quantum_bf16(o) / 2).clamp_min(0) - 2 * U * f64.abs()).max().item()
    print(f'silu: max |fast-math silu - silu| beyond 2u|silu| <= {err:.3g} (SILU_ABS {SILU_ABS:.3g})')
    check('silu', 'silu forward on every bf16 input', out, v, a)
    c = 2048
    yg = every_bf16(c)
    saved = torch.stack([torch.zeros(c, device='cuda'), torch.ones(c, device='cuda')])
    ss = torch.stack([torch.ones(c, device='cuda'), torch.zeros(c, device='cuda')])
    one = torch.ones(1, c, device='cuda', dtype=torch.bfloat16)
    got = torch.empty(yg.shape, device='cuda')
    for i in range(yg.shape[0]):
        sums = nan(2, c)
        ops.bn_bwd_reduce(one, None, yg[i:i + 1].contiguous(), saved, sums, 3, scale_shift=ss)
        got[i] = sums[0]
    f, a = _silu_grad64(yg.double())
    err = ((got.double() - f).abs() - 4 * U * torch.sigmoid(yg.double()) * (1 + yg.double().abs())).max().item()
    print(f"silu': max |fast-math silu' - silu'| beyond its roundings ~ {err:.3g} (SILU_ABS {SILU_ABS:.3g})")
    check('silu', "silu' on every bf16 input", got, f, a)


# ------------------------------------------------------------------ slab BatchNorm: geometry
SLAB_C = [64, 128, 160, 256, 320, 512, 1024, 2048]
ACTS = [0, 1, 2, 3, 1 | 8, 2 | 8]
RES = ['none', 'plain', 'bn']


def _slab_rows(c):
    q = _slab(1, c, 8)[0] * 8 * PARTIAL_ROWS       # a multiple of the stats slab that fills all 264 partial rows
    return [2, 7, q - 1, q + 1, 50176]


GEOM = [(c, rows) for c in SLAB_C for rows in _slab_rows(c)]


def _geom_mode(i, c):
    act, res = ACTS[i % len(ACTS)], RES[(i // 2) % len(RES)]
    if act == 1 and c % 32 == 0:
        src = 'bits' if i % 4 < 2 else 'out'
    else:
        src = 'recompute' if act else 'none'
    return act, res, src


@pytest.mark.parametrize('c,rows', GEOM + [(64, 3211264)])
def test_slab_bn_geometry_conforms(c, rows):
    """Every slab geometry branch: vectors per row a power of two or not (160, 320), ty_count == 1 (2048), one block,
    a slab multiple +- 1 (a ragged last slab), and ResNet-50's stem at batch 256 (3 211 264 x 64).  The activation,
    residual and mask source rotate over the cases; test_slab_bn_modes_conform covers every combination."""
    i = GEOM.index((c, rows)) if (c, rows) in GEOM else 1
    act, res, src = _geom_mode(i, c)
    what = f'bn rows {rows} c {c} act {act} res {res}'
    inputs, outs = _run_slab_bn(rows, c, act, res, [src], seed=100 + i, accumulate=(i % 2 == 1,), what=what)
    _check_slab_bn('slab bn', what, inputs, outs, rows, c, act)
    # invariants: partial_rows = 0 against the mirror's count, and a second launch of the whole chain
    y, gamma, beta, rm0, rv0 = inputs[:5]
    explicit = _bn_forward(y, gamma, beta, 1e-5, 0.1, rm0, rv0, partial_rows=_slab(rows, c, 8)[2])
    _same_all(f'{what} finalize(partial_rows={_slab(rows, c, 8)[2]})', outs['fwd'], explicit)
    if rows < 3211264:
        _, again = _run_slab_bn(rows, c, act, res, [src], seed=100 + i, accumulate=(i % 2 == 1,))
        a, b = _flatten(outs), _flatten(again)
        for k in a:
            if a[k] is not None:
                same(f'{what} {k} on a second launch', a[k], b[k])


def _sources(act, c):
    if act == 0:
        return ['none']
    if act & 8:
        return ['recompute']          # the runtime's path: the mask of act(bn(y)) comes from y
    if act == 3:
        return ['recompute']          # the C ABI refuses SiLU from `out`
    if act == 1 and c % 32 == 0:
        return ['out', 'bits', 'recompute']
    return ['out', 'recompute']


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('res', RES)
@pytest.mark.parametrize('c,rows', [(256, 1000), (160, 999)])
def test_slab_bn_modes_conform(c, rows, act, res):
    """Every activation (ReLU, LeakyReLU 0.1, SiLU, and the DarkNet form act(bn(y)) + res), residual (none, plain,
    batch-normalised by res_scale_shift), every mask source the C ABI allows for it, and dgamma / dbeta written and
    accumulated."""
    what = f'bn modes c {c} act {act} res {res}'
    inputs, outs = _run_slab_bn(rows, c, act, res, _sources(act, c), seed=300 + act * 7 + RES.index(res),
                                accumulate=(False, True), what=what)
    _check_slab_bn('slab bn modes', what, inputs, outs, rows, c, act)


@pytest.mark.parametrize('rows,c', [(3000, 256), (98, 2048), (1001, 160)])
@pytest.mark.parametrize('masked', [True, False])
def test_two_bn_backward_conforms(rows, c, masked):
    """bn_bwd_reduce2 / bn_bwd_apply2 (bn3 and the downsample BatchNorm of one gradient) against the float64 backward;
    their bit equality with two single calls is test_mask_bits_gpu.py's."""
    if masked and c % 32:
        pytest.skip('mask bits need c % 32 == 0')
    ya, ga, ba, _, _ = _bn_case(rows, c, 500)
    yb, gb, bb, _, _ = _bn_case(rows, c, 510)
    fa = _bn_forward(ya, ga, ba, 1e-5, 0.1, None, None)
    fb = _bn_forward(yb, gb, bb, 1e-5, 0.1, None, None)
    out, bits = torch.full_like(ya, NAN), (ops.mask_bits_like(ya) if masked else None)
    ops.bn_apply(ya, fa['ss'], out, 1, res=yb, res_scale_shift=fb['ss'], mask_bits=bits)
    dout = randn(rows, c, seed=520).to(torch.bfloat16)
    prev = [(randn(c, seed=530 + k), randn(c, seed=540 + k)) for k in range(2)]

    def run():
        sums = nan(4, c)
        ws = ops.partial_ws(ya.device, 4 * c)
        ws.fill_(NAN)
        ops.bn_bwd_reduce2(dout, bits, ya, yb, fa['saved'], fb['saved'], sums)
        o = {'sums': sums, 'dya': torch.full_like(ya, NAN), 'dyb': torch.full_like(yb, NAN),
             'dga': nan(c), 'dba': nan(c), 'dgb': prev[1][0].clone(), 'dbb': prev[1][1].clone()}
        ops.bn_bwd_apply2(dout, bits, ya, yb, fa['saved'], fb['saved'], ga, gb, sums, o['dya'], o['dyb'], o['dga'],
                          o['dba'], o['dgb'], o['dbb'], accumulate_a=False, accumulate_b=True)
        return o

    o = run()
    f = _unpack_bits(bits, c) if masked else 1.0
    depth = _slab_depth(rows, c, 4)
    what = f'two-bn rows {rows} c {c}{" bits" if masked else ""}'
    _check_bwd('two-bn backward', what + ' A', dout, ya, fa['saved'], ga, f, 0.0,
               {'sums': o['sums'][:2], 'dy': o['dya'], 'dgamma': o['dga'], 'dbeta': o['dba']}, depth)
    _check_bwd('two-bn backward', what + ' B', dout, yb, fb['saved'], gb, f, 0.0,
               {'sums': o['sums'][2:], 'dy': o['dyb'], 'dgamma': o['dgb'], 'dbeta': o['dbb']}, depth, prev=prev[1])
    _same_all(what, o, run())


# ------------------------------------------------------------------ statistics with an offset
def _torch_rstd(x):
    _, _, invstd = torch.ops.aten.native_batch_norm(x.float(), None, None, None, None, True, 0.1, 1e-5)
    return invstd


@pytest.mark.parametrize('offset', [0, 8, 64])
def test_slab_bn_offset_statistics(offset):
    """|mean| / std up to `offset` per channel, bf16 input: the one-pass variance against its stated allowance, and the
    backward's B y + K cancellation.  Prints the relative rstd error next to torch's fp32 batch_norm."""
    rows, c = 25088, 128
    y, gamma, beta, rm0, rv0 = _bn_case(rows, c, 600 + offset, offset=float(offset))
    fo = _bn_forward(y, gamma, beta, 1e-5, 0.1, rm0, rv0)
    what = f'slab bn offset {offset}'
    r, _ = _check_finalize('slab bn offset', what, y, gamma, beta, 1e-5, 0.1, rm0, rv0, fo, _slab_depth(rows, c, 8))
    ours = ((fo['saved'][1].double() - r).abs() / r).max().item()
    theirs = ((_torch_rstd(y).double() - r).abs() / r).max().item()
    print(f'{what}: max relative rstd error {ours:.3g} (torch fp32 batch_norm: {theirs:.3g})')
    dout = randn(rows, c, seed=610).to(torch.bfloat16)
    o = _bn_backward(dout, y, fo['saved'], gamma, None, 0, 'none', None, None, want_dres=False)
    _check_bwd('slab bn offset', what + ' bwd', dout, y, fo['saved'], gamma, 1.0, 0.0, o, _slab_depth(rows, c, 4))


@pytest.mark.parametrize('offset', [0, 64, 512])
def test_generic_bn_offset_statistics(offset):
    """The generic BatchNorm's statistics of an fp32 stream (VAN) with |mean| / std up to `offset`."""
    rows, c = 6272, 96
    std = rand(c, seed=620) * 1.5 + 0.5
    mean = (rand(c, seed=621) * 2 - 1) * offset * std
    x = randn(rows, c, seed=622) * std + mean
    gamma, beta = randn(c, seed=623) * 0.5 + 1, randn(c, seed=624) * 0.5
    ws = ops.partial_ws(x.device, 2 * c)
    ws.fill_(NAN)
    part, nrows = ops.bn_stats_generic(x)
    fo = {'ss': nan(2, c), 'saved': nan(2, c)}
    ops.bn_finalize(part, gamma, beta, None, None, fo['ss'], fo['saved'], rows, 1e-5, 0.1, partial_rows=nrows)
    ty, rpb, nblk = van_slab(rows, c)
    what = f'generic bn offset {offset}'
    r, _ = _check_finalize('generic bn offset', what, x, gamma, beta, 1e-5, 0.1, None, None, fo,
                           -(-rpb // ty) + ty + -(-nblk // 32) + 32)
    ours = ((fo['saved'][1].double() - r).abs() / r).max().item()
    theirs = ((_torch_rstd(x).double() - r).abs() / r).max().item()
    print(f'{what}: max relative rstd error {ours:.3g} (torch fp32 batch_norm: {theirs:.3g})')


# ------------------------------------------------------------------ generic BatchNorm
@pytest.mark.parametrize('c', [96, 160, 320, 3072])
@pytest.mark.parametrize('x_f32,g_f32,dx_f32', [(a, b, d) for a in (False, True) for b in (False, True) for d in (False, True)])
@pytest.mark.parametrize('with_dres', [False, True])
def test_generic_bn_conforms(c, x_f32, g_f32, dx_f32, with_dres):
    """saicv_bn_*_generic over every dtype combination of x / g / dx; C = 3072 makes each thread loop over two vectors."""
    rows = 6272 if c < 3072 else 1000
    seed = 700 + c
    x = randn(rows, c, seed=seed) * 1.5 + 0.3
    x = x if x_f32 else x.to(torch.bfloat16)
    g = randn(rows, c, seed=seed + 1)
    g = g if g_f32 else g.to(torch.bfloat16)
    dres = randn(rows, c, seed=seed + 2) if with_dres else None
    gamma, beta = randn(c, seed=seed + 3) * 0.5 + 1, randn(c, seed=seed + 4) * 0.5
    ty, rpb, nblk = van_slab(rows, c)
    what = f'generic bn c {c} x {"f32" if x_f32 else "bf16"} g {"f32" if g_f32 else "bf16"} dx {"f32" if dx_f32 else "bf16"}'

    def run():
        ws = ops.partial_ws(x.device, 2 * c)
        ws.fill_(NAN)
        part, nrows = ops.bn_stats_generic(x)
        assert nrows == nblk
        o = {'ss': nan(2, c), 'saved': nan(2, c)}
        ops.bn_finalize(part, gamma, beta, None, None, o['ss'], o['saved'], rows, 1e-5, 0.1, partial_rows=nrows)
        o['out'] = ops.bn_apply_generic(x, o['ss'], dx_f32)
        o['dgamma'], o['dbeta'] = nan(c), nan(c)
        ws.fill_(NAN)
        o['dx'] = ops.bn_bwd_generic(x, g, o['saved'], gamma, o['dgamma'], o['dbeta'], dres=dres, dx_f32=dx_f32)
        return o

    o = run()
    _check_finalize('generic bn stats', what, x, gamma, beta, 1e-5, 0.1, None, None, o, -(-rpb // ty) + ty + -(-nblk // 32) + 32)
    v = x.double() * o['ss'][0].double() + o['ss'][1].double()
    check('generic bn apply', f'{what} apply', o['out'], v, U * v.abs())
    # backward: sums through reduce_partials (sequential over the partial rows)
    n = rows
    depth = -(-rpb // ty) + ty + nblk
    mean, rstd = o['saved'][0].double(), o['saved'][1].double()
    g64 = g.double()
    xh = (x.double() - mean) * rstd
    t1 = g64 * xh
    a0 = (depth + 1) * U * g64.abs().sum(0)
    a1 = (depth + 1) * U * t1.abs().sum(0) + 2 * U * t1.abs().sum(0)
    check('generic bn backward', f'{what} dbeta', o['dbeta'], g64.sum(0), a0)
    check('generic bn backward', f'{what} dgamma', o['dgamma'], t1.sum(0), a1)
    k1 = gamma.double() * rstd
    m0, m1 = o['dbeta'].double() / n, o['dgamma'].double() / n
    inner = g64 - m0 - xh * m1
    v = k1 * inner
    # xhat (2u), sum * (1 / rows) (2u), xhat * sum * (1 / rows) (+3u), two subtractions, gamma * rstd and the product
    a = k1.abs() * 8 * U * (g64.abs() + m0.abs() + (xh * m1).abs()) + 2 * U * v.abs()
    if dres is not None:
        v = v + dres.double()
        a = rnd(v, a)
    check('generic bn backward', f'{what} dx', o['dx'], v, a)
    _same_all(what, o, run())


# ------------------------------------------------------------------ LayerNorm (ViT) and post-LN (DETR)
def _ln_fwd_ref(x64, gamma, beta, eps):
    """Exact LayerNorm of x64 [rows, C]; allowances of the kernel's mean, rstd and normalised output."""
    rows, c = x64.shape
    depth = 4 * (c // 128) + 5                      # per-lane chain of 4-element adds + the warp butterfly
    mean = x64.mean(1, keepdim=True)
    xc = x64 - mean
    var = (xc * xc).mean(1, keepdim=True)
    e0 = (depth + 1) * U * x64.abs().mean(1, keepdim=True)
    a_m = e0 + 3 * U * (mean.abs() + e0)
    a_q = (depth + 4) * U * var + a_m * a_m + 2 * a_m * xc.mean(1, keepdim=True).abs()
    a_v = a_q + 3 * U * (var + a_q)
    r, a_r = _rstd_interval(var, a_v, eps)
    g, b = gamma.double(), beta.double()
    t = xc * r * g
    y = t + b
    a_y = g.abs() * (xc.abs() * a_r + (r + a_r) * a_m) + 4 * U * (t.abs() + b.abs())
    return mean.squeeze(1), a_m.squeeze(1), r.squeeze(1), a_r.squeeze(1), y, a_y


def _ln_bwd_ref(dy64, x64, gamma, stats):
    """Exact LayerNorm data gradient from the kernel's saved (mean, rstd), with its allowance, and the parameter-gradient
    terms dy * xhat."""
    rows, c = x64.shape
    depth = 4 * (c // 128) + 5
    mean, rstd = stats[0].double()[:, None], stats[1].double()[:, None]
    xh = (x64 - mean) * rstd
    d = dy64 * gamma.double()
    c1 = d.mean(1, keepdim=True)
    a_c1 = (depth + 2) * U * d.abs().mean(1, keepdim=True) + 2 * U * c1.abs()
    dx = d * xh
    c2 = dx.mean(1, keepdim=True)
    a_c2 = (depth + 5) * U * dx.abs().mean(1, keepdim=True) + 2 * U * c2.abs()
    inner = d - c1 - xh * c2
    v = rstd * inner
    a = rstd * (U * d.abs() + a_c1 + xh.abs() * a_c2 + 2 * U * xh.abs() * c2.abs()
                + 3 * U * (d.abs() + c1.abs() + (xh * c2).abs())) + U * v.abs()
    return v, a, xh


def _check_param_grads(fam, what, dy64, xh, o, depth, prev=None):
    tb, tg = dy64, dy64 * xh
    for name, t, k in (('dbeta', tb, 1), ('dgamma', tg, 0)):
        s = t.sum(0)
        a = (depth + 1) * U * t.abs().sum(0) + (3 * U * t.abs().sum(0) if name == 'dgamma' else 0.0)
        if prev is not None:
            s = prev[k].double() + s
            a = rnd(s, a)
        check(fam, f'{what} {name}{" (accumulate)" if prev is not None else ""}', o[name], s, a)


LN_C = [128, 256, 384, 512, 768, 1024, 1280]
LN_ROWS = [1, 7, 2113, 50432]      # 2113: more rows than the forward's 132 * 8 blocks of 8 warps


@pytest.mark.parametrize('c', LN_C)
@pytest.mark.parametrize('rows', LN_ROWS)
@pytest.mark.parametrize('eps', [1e-6, 1e-5])
def test_layernorm_conforms(c, rows, eps):
    """saicv_layernorm_fwd / _bwd at every compiled width.  The backward runs twice: plain into fresh dgamma / dbeta,
    then with the residual-stream gradient dres, the bf16 copy scaled per 197 rows by a drop-path scale, accumulating
    onto the first call's parameter gradients."""
    seed = 800 + c + rows
    x = randn(rows, c, seed=seed) * 2 + (randn(c, seed=seed + 1) * 0.5)
    gamma, beta = randn(c, seed=seed + 2) * 0.5 + 1, randn(c, seed=seed + 3) * 0.5
    dy = randn(rows, c, seed=seed + 4).to(torch.bfloat16)
    dres = randn(rows, c, seed=seed + 5)
    rps = 197
    scale = (rand(-(-rows // rps), seed=seed + 6) > 0.3).float() * 1.25
    what = f'ln rows {rows} c {c} eps {eps:g}'

    def run():
        o = {'y': torch.full((rows, c), NAN, device='cuda', dtype=torch.bfloat16), 'stats': nan(2, rows)}
        ops.layernorm_fwd(x, gamma, beta, eps, out=o['y'], stats=o['stats'])
        o['dgamma'], o['dbeta'] = nan(c), nan(c)
        o['dx'] = ops.layernorm_bwd(dy, x, gamma, o['stats'], o['dgamma'], o['dbeta'], dx=nan(rows, c))
        o['dgamma1'], o['dbeta1'] = o['dgamma'].clone(), o['dbeta'].clone()
        o['dxb'] = torch.full((rows, c), NAN, device='cuda', dtype=torch.bfloat16)
        o['dx2'] = ops.layernorm_bwd(dy, x, gamma, o['stats'], o['dgamma1'], o['dbeta1'], dres=dres, dx=nan(rows, c),
                                     dx_bf16=o['dxb'], accumulate=True, bf16_row_scale=scale, rows_per_scale=rps)
        return o

    o = run()
    x64 = x.double()
    mean, a_m, r, a_r, y, a_y = _ln_fwd_ref(x64, gamma, beta, eps)
    check('layernorm fwd', f'{what} mean', o['stats'][0], mean, a_m)
    check('layernorm fwd', f'{what} rstd', o['stats'][1], r, a_r)
    check('layernorm fwd', f'{what} y', o['y'], y, a_y)
    del y, a_y
    dy64 = dy.double()
    v, a, xh = _ln_bwd_ref(dy64, x64, gamma, o['stats'])
    check('layernorm bwd', f'{what} dx', o['dx'], v, a)
    depth = _ln_bwd_depth(rows)
    _check_param_grads('layernorm bwd', what, dy64, xh, o, depth)
    v = v + dres.double()
    a = rnd(v, a)
    check('layernorm bwd', f'{what} dx + dres', o['dx2'], v, a)
    sc = scale.double().repeat_interleave(rps)[:rows, None]
    check('layernorm bwd', f'{what} bf16 dx * drop-path scale', o['dxb'], v * sc, a * sc + U * (v * sc).abs())
    _check_param_grads('layernorm bwd', what, dy64, xh, {'dgamma': o['dgamma1'], 'dbeta': o['dbeta1']},
                       _ln_bwd_depth(rows, True), prev=(o['dgamma'], o['dbeta']))
    del v, a, xh
    _same_all(what, o, run())


POSTLN = [(c, rows, pr) for c in (128, 256, 384, 512) for rows, pr in ((2 * 850, 850), (850, 850), (6 * 100, 100))]


@pytest.mark.parametrize('c,rows,pos_rows', POSTLN)
def test_postln_conforms(c, rows, pos_rows):
    """saicv_postln_fwd / _bwd (DETR): y fp32, its bf16 copy, bf16(y + pos[row % pos_rows]) with pos_rows dividing rows
    or equal to it; the backward with dres and both outputs; add_pos_cast."""
    seed = 900 + c + rows
    z = randn(rows, c, seed=seed) * 3
    gamma, beta = randn(c, seed=seed + 1) * 0.5 + 1, randn(c, seed=seed + 2) * 0.5
    pos = randn(pos_rows, c, seed=seed + 3)
    dy = randn(rows, c, seed=seed + 4)
    dres = randn(rows, c, seed=seed + 5)
    prev = (randn(c, seed=seed + 6), randn(c, seed=seed + 7))
    what = f'postln rows {rows} c {c} pos_rows {pos_rows}'

    def run():
        y, yb, ypb, stats = ops.postln_fwd(z, gamma, beta, 1e-5, pos=pos, want_y=True, want_yb=True, want_ypb=True)
        dg, db = prev[0].clone(), prev[1].clone()
        dz, dzb = ops.postln_bwd(dy, z, gamma, stats, dg, db, dres=dres, accumulate=True)
        xb, xpb = ops.add_pos_cast(z, pos)
        return {'y': y, 'yb': yb, 'ypb': ypb, 'stats': stats, 'dz': dz, 'dzb': dzb, 'dgamma': dg, 'dbeta': db,
                'xb': xb, 'xpb': xpb}

    o = run()
    z64 = z.double()
    mean, a_m, r, a_r, y, a_y = _ln_fwd_ref(z64, gamma, beta, 1e-5)
    check('postln fwd', f'{what} mean', o['stats'][0], mean, a_m)
    check('postln fwd', f'{what} rstd', o['stats'][1], r, a_r)
    check('postln fwd', f'{what} y', o['y'], y, a_y)
    check('postln fwd', f'{what} yb', o['yb'], y, a_y)
    p64 = pos.double().repeat(rows // pos_rows, 1)
    yp = y + p64
    check('postln fwd', f'{what} ypb', o['ypb'], yp, rnd(yp, a_y))
    del y, a_y, yp
    dy64 = dy.double()
    v, a, xh = _ln_bwd_ref(dy64, z64, gamma, o['stats'])
    v = v + dres.double()
    a = rnd(v, a)
    check('postln bwd', f'{what} dz', o['dz'], v, a)
    check('postln bwd', f'{what} dzb', o['dzb'], v, a)
    _check_param_grads('postln bwd', what, dy64, xh, o, _ln_bwd_depth(rows, True), prev=prev)
    same('add_pos_cast xb', o['xb'], z.to(torch.bfloat16))
    zp = z64 + p64
    check('add_pos_cast', f'{what} add_pos_cast xpb', o['xpb'], zp, U * zp.abs())
    _same_all(what, o, run())


@pytest.mark.parametrize('want_y,want_yb,want_ypb', [(a, b, d) for a in (False, True) for b in (False, True) for d in (False, True)])
@pytest.mark.parametrize('want_dz,want_dzb', [(False, False), (False, True), (True, False), (True, True)])
def test_postln_nullable_outputs(want_y, want_yb, want_ypb, want_dz, want_dzb):
    """Every nullable output combination writes what the full call writes, bit for bit (and add_pos_cast's)."""
    rows, c, pos_rows = 300, 256, 100
    z = randn(rows, c, seed=950) * 3
    gamma, beta = randn(c, seed=951) * 0.5 + 1, randn(c, seed=952) * 0.5
    pos = randn(pos_rows, c, seed=953)
    dy = randn(rows, c, seed=954)
    y0, yb0, ypb0, st0 = ops.postln_fwd(z, gamma, beta, 1e-5, pos=pos, want_y=True, want_yb=True, want_ypb=True)
    y, yb, ypb, st = ops.postln_fwd(z, gamma, beta, 1e-5, pos=pos, want_y=want_y, want_yb=want_yb, want_ypb=want_ypb)
    same('stats', st, st0)
    for name, a, b in (('y', y, y0), ('yb', yb, yb0), ('ypb', ypb, ypb0)):
        assert (a is not None) == {'y': want_y, 'yb': want_yb, 'ypb': want_ypb}[name]
        if a is not None:
            same(name, a, b)
    dg0, db0, dg, db = nan(c), nan(c), nan(c), nan(c)
    dz0, dzb0 = ops.postln_bwd(dy, z, gamma, st0, dg0, db0)
    dz, dzb = ops.postln_bwd(dy, z, gamma, st0, dg, db, want_dz=want_dz, want_dzb=want_dzb)
    same('dgamma', dg, dg0)
    same('dbeta', db, db0)
    if want_dz:
        same('dz', dz, dz0)
    if want_dzb:
        same('dzb', dzb, dzb0)
    xb0, xpb0 = ops.add_pos_cast(z, pos)
    xb, xpb = ops.add_pos_cast(z, pos, want_xb=want_y, want_xpb=want_yb)
    if want_y:
        same('xb', xb, xb0)
    if want_yb:
        same('xpb', xpb, xpb0)


# ------------------------------------------------------------------ column sums
@pytest.mark.parametrize('c', [8, 768, 2048, 2056, 3072, 4104])
@pytest.mark.parametrize('accumulate', [False, True])
def test_colsum_conforms(c, accumulate):
    """bf16 column sums in chunks of at most 2048 columns (2056 and 4104 leave an 8-column chunk)."""
    rows = 20000
    x = randn(rows, c, seed=1000 + c).to(torch.bfloat16)
    prev = randn(c, seed=1001)

    def run():
        out = prev.clone() if accumulate else nan(c)
        ops.partial_ws(x.device, c).fill_(NAN)
        return {'out': ops.colsum(x, out, accumulate=accumulate)}

    o = run()
    x64 = x.double()
    s, a = x64.sum(0), torch.empty(c, device='cuda', dtype=torch.float64)
    for c0 in range(0, c, 2048):
        cw = min(2048, c - c0)
        a[c0:c0 + cw] = (_slab_depth(rows, cw, 8) + 1) * U * x64[:, c0:c0 + cw].abs().sum(0)
    if accumulate:
        s = prev.double() + s
        a = rnd(s, a)
    check('colsum', f'colsum c {c} rows {rows}{" accumulate" if accumulate else ""}', o['out'], s, a)
    _same_all(f'colsum c {c}', o, run())


@pytest.mark.parametrize('rows,c', [(256, 1000), (50, 4104)])
@pytest.mark.parametrize('accumulate', [False, True])
def test_colsum_f32_conforms(rows, c, accumulate):
    x = randn(rows, c, seed=1100 + c)
    prev = randn(c, seed=1101)

    def run():
        out = prev.clone() if accumulate else nan(c)
        return {'out': ops.colsum(x, out, accumulate=accumulate)}

    o = run()
    x64 = x.double()
    s, a = x64.sum(0), (rows + 1) * U * x64.abs().sum(0)
    if accumulate:
        s = prev.double() + s
        a = rnd(s, a)
    check('colsum f32', f'colsum f32 rows {rows} c {c}', o['out'], s, a)
    _same_all('colsum f32', o, run())


# ------------------------------------------------------------------ pooling
def _maxpool_ref(x, k, stride, pad, pad_hi, oob_zero):
    """float64 max-pool with torch's tie rule: value and argmax code (r * k + s, or 255 for a zero-padded tap)."""
    n, h, w, c = x.shape
    xp = F.pad(x.double().permute(0, 3, 1, 2), (pad, pad_hi, pad, pad_hi), value=0.0 if oob_zero else float('-inf'))
    inside = F.pad(torch.ones(1, 1, h, w, device='cuda', dtype=torch.float64), (pad, pad_hi, pad, pad_hi))
    P, Q = (h + pad + pad_hi - k) // stride + 1, (w + pad + pad_hi - k) // stride + 1
    kk = k * k
    cols = F.unfold(xp, k, stride=stride).view(n, c, kk, P * Q)
    ins = F.unfold(inside, k, stride=stride).view(1, 1, kk, P * Q) > 0
    m = cols.max(2, keepdim=True).values
    first = ((cols == m) * torch.arange(kk, 0, -1, device='cuda').view(1, 1, kk, 1)).argmax(2, keepdim=True)
    code = torch.where(torch.gather(ins.expand(n, c, kk, P * Q), 2, first), first, 255)
    to_nhwc = lambda t: t.view(n, c, P, Q).permute(0, 2, 3, 1)
    return to_nhwc(m), to_nhwc(code), P, Q


def _maxpool_bwd_ref(dy, code, h, w, k, stride, pad, pad_hi):
    n, P, Q, c = dy.shape
    kk = k * k
    g = dy.double().permute(0, 3, 1, 2).reshape(n, c, 1, P * Q)
    t = code.permute(0, 3, 1, 2).reshape(n, c, 1, P * Q).long()
    hit = (t == torch.arange(kk, device='cuda').view(1, 1, kk, 1)).double()
    size = (h + pad + pad_hi, w + pad + pad_hi)
    fold = lambda v: F.fold((v * hit).view(n, c * kk, P * Q), size, k, stride=stride)[:, :, pad:pad + h, pad:pad + w]
    return fold(g).permute(0, 2, 3, 1), fold(g.abs()).permute(0, 2, 3, 1)


@pytest.mark.parametrize('n,h,w,c,k,stride,pad,pad_hi,oob_zero', [
    (2, 112, 112, 64, 3, 2, 1, 1, 0),      # ResNet stem pool
    (3, 9, 9, 24, 3, 2, 1, 1, 0),
    (3, 7, 7, 24, 3, 2, 1, 1, 0),
    (2, 8, 10, 16, 2, 2, 0, 0, 0),
    (2, 13, 13, 16, 2, 1, 0, 1, 1),        # DarkNet-tiny ZeroPad2d((0, 1, 0, 1)) + MaxPool2d(2, 1)
    (2, 9, 9, 16, 3, 1, 1, 1, 0),          # non-FAST backward
    (2, 9, 11, 16, 5, 1, 2, 2, 0),         # runtime-K forward, non-FAST backward
])
def test_maxpool_conforms(n, h, w, c, k, stride, pad, pad_hi, oob_zero):
    """Inputs are ReLU outputs of a few bf16 values: most windows hold ties and some are all zero, so the tie rule
    decides the argmax, and with it which input receives the gradient."""
    vals = torch.tensor([-1.0, -0.5, 0.0, 0.5, 1.0, 0.5, 0.0], device='cuda')
    idx = torch.randint(0, vals.numel(), (n, h, w, c), device='cuda', generator=gen(1200 + k + h))
    x = vals[idx].clamp_min(0).to(torch.bfloat16)
    P, Q = (h + pad + pad_hi - k) // stride + 1, (w + pad + pad_hi - k) // stride + 1
    dy = randn(n, P, Q, c, seed=1201).to(torch.bfloat16)

    def run():
        y, am = ops.maxpool_fwd(x, k, stride, pad, pad_hi, bool(oob_zero))
        return {'y': y, 'argmax': am, 'dx': ops.maxpool_bwd(dy, am, h, w, k, stride, pad, pad_hi)}

    o = run()
    m, code, P2, Q2 = _maxpool_ref(x, k, stride, pad, pad_hi, oob_zero)
    assert (P2, Q2) == (P, Q)
    what = f'maxpool {k}x{k}/{stride} pad {pad},{pad_hi}{" zero" if oob_zero else ""} {n}x{h}x{w}x{c}'
    ties = ((F.unfold(F.pad(x.double().permute(0, 3, 1, 2), (pad, pad_hi, pad, pad_hi)), k, stride=stride)
             .view(n, c, k * k, -1) == m.permute(0, 3, 1, 2).reshape(n, c, 1, -1)).sum(2) > 1).double().mean().item()
    print(f'{what}: {ties:.0%} of the windows have a tied maximum')
    n_bad = int((o['y'].double() != m).sum())
    assert n_bad == 0, f'{what}: {n_bad} pooled values differ'
    n_bad = int((o['argmax'].long() != code).sum())
    assert n_bad == 0, f'{what}: {n_bad} argmax codes differ from the first maximum in scan order'
    v, s = _maxpool_bwd_ref(dy, code, h, w, k, stride, pad, pad_hi)
    check('maxpool bwd', f'{what} dx', o['dx'], v, (-(-k // stride)) ** 2 * U * s)
    _same_all(what, o, run())
    if (k, stride, pad, pad_hi, oob_zero) == (3, 2, 1, 1, 0):     # the ResNet stem pool's own entries
        y, am = ops.maxpool3x3s2_fwd(x)
        stem = {'y': y, 'argmax': am, 'dx': ops.maxpool3x3s2_bwd(dy, am, h, w)}
        for key in o:
            same(f'{what}: maxpool3x3s2 {key}', stem[key], o[key])


@pytest.mark.parametrize('n,h,w,c', [(8, 7, 7, 2048), (4, 14, 14, 512), (3, 1, 1, 64)])
def test_avgpool_conforms(n, h, w, c):
    x = (randn(n, h, w, c, seed=1300) + 0.5).to(torch.bfloat16)
    dy = randn(n, c, seed=1301).to(torch.bfloat16)

    def run():
        return {'y': ops.avgpool_fwd(x), 'dx': ops.avgpool_bwd(dy, h, w)}

    o = run()
    hw = h * w
    x64 = x.double().view(n, hw, c)
    v = x64.sum(1) / hw
    a = rnd(v, rnd(v, hw * U * x64.abs().sum(1) / hw))      # hw - 1 adds, then 1 / hw and the product round
    check('avgpool', f'avgpool fwd {n}x{h}x{w}x{c}', o['y'], v, a)
    vb = (dy.double() / hw)[:, None, None, :].expand(n, h, w, c)
    check('avgpool', f'avgpool bwd {n}x{h}x{w}x{c}', o['dx'], vb, 2 * U * vb.abs())
    _same_all('avgpool', o, run())


@pytest.mark.parametrize('x_f32', [False, True])
@pytest.mark.parametrize('dx_f32', [False, True])
def test_avgpool_stream_conforms(x_f32, dx_f32):
    n, h, w, c = 4, 7, 7, 512
    x = randn(n, h, w, c, seed=1400) + 0.5
    x = x if x_f32 else x.to(torch.bfloat16)
    dy = randn(n, c, seed=1401).to(torch.bfloat16)

    def run():
        return {'y': ops.avgpool_stream_fwd(x), 'dx': ops.avgpool_stream_bwd(dy, h, w, dx_f32=dx_f32)}

    o = run()
    hw = h * w
    x64 = x.double().view(n, hw, c)
    v = x64.sum(1) / hw
    a = rnd(v, rnd(v, hw * U * x64.abs().sum(1) / hw))      # hw - 1 adds, then 1 / hw and the product round
    what = f'avgpool_stream x {"f32" if x_f32 else "bf16"} dx {"f32" if dx_f32 else "bf16"}'
    check('avgpool stream', f'{what} fwd', o['y'], v, a)
    vb = (dy.double() / hw)[:, None, None, :].expand(n, h, w, c)
    check('avgpool stream', f'{what} bwd', o['dx'], vb, 2 * U * vb.abs())
    _same_all(what, o, run())
