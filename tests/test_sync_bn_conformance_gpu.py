"""Conformance of the synchronized-BatchNorm kernels (cross-rank statistics) against a float64 reference, and their
bit-identity invariants.

A [rows, C] activation is split into W "virtual ranks" of unequal row counts.  Each part is folded on its own
(saicv_bn_stats_fold over the partials of bn_stats, bn_stats_generic or the GEMM epilogue), and the folded buffers are
summed on the device in fp32, which is what the all-reduce of the runtime computes.  Then finalize, apply, the
backward reduce of each part, the same sum of the backward sums, and the backward apply with the global sums, the
part's own sums (dgamma / dbeta) and the global row count.  Everything is compared with float64 BatchNorm over the
concatenated rows, under the allowances of tests/conformance.py (u = 2^-24 per fp32 rounding, derived, never fitted):
  * a fold of depth d_k per part (the mirrors of slab_geom / van slab below) plus W - 1 fp32 additions across parts is
    a reduction of depth max d_k + W - 1 over all rows;
  * mean, one-pass variance, rstd, scale / shift and running statistics then carry the allowances of
    test_norm_conformance_gpu.py, with the unbiased variance taken over the GLOBAL row count;
  * dgamma / dbeta of each part are its LOCAL sums (depth d_k); dy / dx are checked from the kernel's own summed
    backward sums over the global count, with the allowances of the unsynchronized backward kernels.
Invariants (raw bits): with one part, fold + finalize_folded equals bn_finalize and the _sync / split backward entry
points equal the plain ones; the row count rides in the buffer exactly beyond 2^24 rows.
"""
import math

import pytest
import torch

from conformance import NAN, PARTIAL_ROWS, U, check, exact, nan, next_pow2, rand, randn, rnd, same, van_slab
from conformance import report  # noqa: F401  (autouse: this module's allowance report)

from simpleaicv_pytorch_training_examples_b200 import ops

pytestmark = pytest.mark.gpu

RSQRT = 2.0 ** -22      # rsqrtf: 2 ulp, relative
EPS, MOM = 1e-5, 0.1


# ------------------------------------------------------------------ launch geometry mirrors
def _slab(rows, c, unroll, max_blocks=PARTIAL_ROWS):
    """capi_elementwise.cu slab_geom: (ty_count, rows_per_block, blocks)."""
    tx = min(next_pow2(c // 8), 256)
    ty = 256 // tx
    b = max(1, min(-(-rows // (ty * unroll)), max_blocks))
    q = ty * unroll
    rpb = -(-(-(-rows // b)) // q) * q
    return ty, rpb, -(-rows // rpb)


def _slab_depth(rows, c, unroll):
    ty, rpb, nblk = _slab(rows, c, unroll)
    return -(-rpb // ty) + int(math.log2(ty)) + -(-nblk // 32) + 32


def _generic_stats_depth(rows, c):
    ty, rpb, nblk = van_slab(rows, c)
    return -(-rpb // ty) + ty + -(-nblk // 32) + 32


def _generic_bwd_depth(rows, c):
    ty, rpb, nblk = van_slab(rows, c)
    return -(-rpb // ty) + ty + nblk


# ------------------------------------------------------------------ float64 references
def _stats_allow(x64, depth):
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


def _check_finalize(fam, what, x, gamma, beta, rm0, rv0, o, depth):
    """Finalize outputs o = {ss, saved, rm, rv} against the exact statistics of ALL rows x."""
    n = x.shape[0]
    mean, var, a_m, a_v = _stats_allow(x.double(), depth)
    e = torch.tensor(EPS, dtype=torch.float32).double().item()
    r = (var + e).rsqrt()
    t_lo = ((var - a_v).clamp_min(0) + e) * (1 - 2 * U)
    t_hi = (var + a_v + e) * (1 + 2 * U)
    a_r = torch.maximum(t_lo.rsqrt() * (1 + RSQRT) - r, r - t_hi.rsqrt() * (1 - RSQRT))
    g, b = gamma.double(), beta.double()
    check(fam, f'{what} mean', o['saved'][0], mean, a_m)
    check(fam, f'{what} rstd', o['saved'][1], r, a_r)
    sc = g * r
    a_sc = g.abs() * a_r + U * g.abs() * (r + a_r)
    sh = b - mean * sc
    a_sh = mean.abs() * a_sc + (sc.abs() + a_sc) * a_m + 2 * U * ((mean.abs() + a_m) * (sc.abs() + a_sc) + b.abs())
    check(fam, f'{what} scale', o['ss'][0], sc, a_sc)
    check(fam, f'{what} shift', o['ss'][1], sh, a_sh)
    rm = (1 - MOM) * rm0.double() + MOM * mean
    a_rm = MOM * a_m + 5 * U * ((1 - MOM) * rm0.double().abs() + MOM * (mean.abs() + a_m))
    unb = n / (n - 1)          # the GLOBAL row count
    rv = (1 - MOM) * rv0.double() + MOM * unb * var
    a_rv = MOM * unb * a_v + 7 * U * ((1 - MOM) * rv0.double().abs() + MOM * unb * (var + a_v))
    check(fam, f'{what} running_mean', o['rm'], rm, a_rm)
    check(fam, f'{what} running_var', o['rv'], rv, a_rv)


def _local_sums_ref(ge, a_ge, y, saved, depth):
    """Exact sum g | sum g * xhat of one part (global mean / rstd as stored) and their allowances."""
    mean, rstd = saved[0].double(), saved[1].double()
    xh = (y.double() - mean) * rstd
    t1 = ge * xh
    a0 = (depth + 1) * U * ge.abs().sum(0) + a_ge.sum(0)
    a1 = (depth + 1) * U * t1.abs().sum(0) + (a_ge * xh.abs() + 3 * U * t1.abs()).sum(0)
    return ge.sum(0), t1.sum(0), a0, a1


def _dy_ref(ge, a_ge, y, saved, gamma, sums, n):
    """bn_bwd_apply's A g + B y + K from the summed (global) sums over the global count n."""
    mean, rstd = saved[0].double(), saved[1].double()
    A = gamma.double() * rstd
    k2, k3 = sums[0].double() / n, sums[1].double() / n
    T1, T2, B = A * k2, A * k3 * rstd * mean, -A * k3 * rstd
    By = B * y.double()
    v = A * ge + By + (T2 - T1)
    return v, A.abs() * a_ge + 10 * U * ((A * ge).abs() + By.abs() + T1.abs() + T2.abs())


# ------------------------------------------------------------------ the virtual ranks
def _split(x, parts):
    out, r0 = [], 0
    for r in parts:
        out.append(x[r0:r0 + r].contiguous())
        r0 += r
    assert r0 == x.shape[0]
    return out


def _allreduce(bufs):
    """The all-reduce stand-in: the sum of the ranks' buffers in fp32, on the device."""
    total = bufs[0].clone()
    for b in bufs[1:]:
        total += b
    return total


def _fold(partials, rows, c, prow):
    stats = ops.bn_stats_fold(partials, rows, c, partial_rows=prow)
    # the count slots hold this part's rows exactly
    assert int(stats[2 * c].item()) * 4096 + int(stats[2 * c + 1].item()) == rows
    return stats


def _case(rows, c, seed, f32=False):
    std = rand(c, seed=seed) * 1.5 + 0.5
    mean = (rand(c, seed=seed + 1) * 2 - 1) * std
    y = randn(rows, c, seed=seed + 2) * std + mean
    y = y if f32 else y.to(torch.bfloat16)
    gamma = randn(c, seed=seed + 3) * 0.5 + 1.0
    beta = randn(c, seed=seed + 4) * 0.5
    rm0, rv0 = randn(c, seed=seed + 5) * 0.1, rand(c, seed=seed + 6) + 0.5
    return y, gamma, beta, rm0, rv0


def _finalize_folded(total, c, gamma, beta, rm0, rv0):
    o = {'ss': nan(2, c), 'saved': nan(2, c), 'rm': rm0.clone(), 'rv': rv0.clone()}
    ops.bn_finalize_folded(total, gamma, beta, o['rm'], o['rv'], o['ss'], o['saved'], EPS, MOM)
    return o


# ------------------------------------------------------------------ convnet path (bn_stats / bn_bwd_reduce / apply)
@pytest.mark.parametrize('c,parts', [(64, (3000, 1000)), (256, (1200, 2500, 700)), (2048, (98, 50)), (512, (3, 5))])
def test_slab_sync_bn_conforms(c, parts):
    """W = len(parts) ranks: statistics, running stats (global unbiased variance), apply with the block-output ReLU mask,
    and the synchronized backward (dy over the global sums and count, dres, local dgamma / dbeta)."""
    rows = sum(parts)
    W = len(parts)
    y, gamma, beta, rm0, rv0 = _case(rows, c, 100 + c)
    dout = randn(rows, c, seed=200 + c).to(torch.bfloat16)
    ys, douts = _split(y, parts), _split(dout, parts)
    stats = []
    for yk in ys:
        ws = ops.partial_ws(y.device, 2 * c)
        ws.fill_(NAN)
        stats.append(_fold(ops.bn_stats(yk, ws), yk.shape[0], c, 0))
    total = _allreduce(stats)
    o = _finalize_folded(total, c, gamma, beta, rm0, rv0)
    what = f'sync bn c {c} parts {parts}'
    depth = max(_slab_depth(r, c, 8) for r in parts) + W - 1
    _check_finalize('sync bn stats', what, y, gamma, beta, rm0, rv0, o, depth)
    # apply (per rank, unchanged kernel) and the packed ReLU mask the backward reads
    outs, bits = [], []
    for yk in ys:
        out, bk = torch.full_like(yk, NAN), ops.mask_bits_like(yk)
        ops.bn_apply(yk, o['ss'], out, 1, mask_bits=bk)
        t = yk.double() * o['ss'][0].double()
        v = t + o['ss'][1].double()
        check('sync bn apply', f'{what} out', out, v.clamp_min(0), 2 * U * (t.abs() + o['ss'][1].double().abs()))
        outs.append(out)
        bits.append(bk)
    # backward: local sums per rank, summed, applied with the global count
    local = []
    for yk, dk, bk in zip(ys, douts, bits):
        s = nan(2, c)
        ops.partial_ws(y.device, 2 * c).fill_(NAN)
        ops.bn_bwd_reduce(dk, None, yk, o['saved'], s, 1, bits=bk)
        local.append(s)
    gsum = _allreduce(local)
    count = ops.bn_sync_count(total, c)
    for k, (yk, dk, bk, outk) in enumerate(zip(ys, douts, bits, outs)):
        dy, dres, dg, db = torch.full_like(yk, NAN), torch.full_like(yk, NAN), nan(c), nan(c)
        ops.bn_bwd_apply(dk, None, yk, o['saved'], gamma, gsum, dy, dres, dg, db, 1, bits=bk,
                         local_sums=local[k], count=count)
        ge = dk.double() * (outk.double() > 0).double()
        a_ge = 2 * U * ge.abs()
        s0, s1, a0, a1 = _local_sums_ref(ge, a_ge, yk, o['saved'], _slab_depth(parts[k], c, 4))
        check('sync bn backward', f'{what} rank {k} dbeta (local)', db, s0, a0)
        check('sync bn backward', f'{what} rank {k} dgamma (local)', dg, s1, a1)
        check('sync bn backward', f'{what} rank {k} dres', dres, ge, a_ge)
        v, a = _dy_ref(ge, a_ge, yk, o['saved'], gamma, gsum, rows)
        check('sync bn backward', f'{what} rank {k} dy', dy, v, a)
    # the summed backward sums against the float64 sums over all rows
    ge = dout.double() * torch.cat([(t.double() > 0).double() for t in outs])
    s0, s1, a0, a1 = _local_sums_ref(ge, 2 * U * ge.abs(), y, o['saved'], max(_slab_depth(r, c, 4) for r in parts) + W - 1)
    check('sync bn backward', f'{what} global sum g', gsum[0], s0, a0)
    check('sync bn backward', f'{what} global sum g*xhat', gsum[1], s1, a1)


@pytest.mark.parametrize('c,parts', [(256, (1500, 900)), (128, (300, 500, 200))])
def test_slab_sync_bn_pair_conforms(c, parts):
    """The paired backward of bn3 and the downsample BatchNorm: one [4, C] exchange, local dgamma / dbeta of both."""
    rows = sum(parts)
    W = len(parts)
    ya, ga, ba, rma, rva = _case(rows, c, 300)
    yb, gb, bb, rmb, rvb = _case(rows, c, 310)
    g = randn(rows, c, seed=320).to(torch.bfloat16)
    fwd = []
    for y, gam, bet, rm, rv in ((ya, ga, ba, rma, rva), (yb, gb, bb, rmb, rvb)):
        st = [_fold(ops.bn_stats(yk), yk.shape[0], c, 0) for yk in _split(y, parts)]
        total = _allreduce(st)
        fwd.append((total, _finalize_folded(total, c, gam, bet, rm, rv)))
    (ta, fa), (_, fb) = fwd
    yas, ybs, gs = _split(ya, parts), _split(yb, parts), _split(g, parts)
    local = []
    for yak, ybk, gk in zip(yas, ybs, gs):
        s = nan(4, c)
        ops.bn_bwd_reduce2(gk, None, yak, ybk, fa['saved'], fb['saved'], s)
        local.append(s)
    gsum = _allreduce(local)
    what = f'sync bn pair c {c} parts {parts}'
    for k, (yak, ybk, gk) in enumerate(zip(yas, ybs, gs)):
        o = {n: torch.full_like(yak, NAN) for n in ('dya', 'dyb')}
        o.update({n: nan(c) for n in ('dga', 'dba', 'dgb', 'dbb')})
        ops.bn_bwd_apply2(gk, None, yak, ybk, fa['saved'], fb['saved'], ga, gb, gsum, o['dya'], o['dyb'], o['dga'],
                          o['dba'], o['dgb'], o['dbb'], local_sums=local[k], count=ops.bn_sync_count(ta, c))
        ge = gk.double()
        for tag, yk, f, gam, sl in (('A', yak, fa, ga, slice(0, 2)), ('B', ybk, fb, gb, slice(2, 4))):
            s0, s1, a0, a1 = _local_sums_ref(ge, 0.0 * ge, yk, f['saved'], _slab_depth(parts[k], c, 4))
            check('sync bn pair', f'{what} rank {k} {tag} dbeta (local)', o['db' + tag.lower()], s0, a0)
            check('sync bn pair', f'{what} rank {k} {tag} dgamma (local)', o['dg' + tag.lower()], s1, a1)
            v, a = _dy_ref(ge, 0.0, yk, f['saved'], gam, gsum[sl], rows)
            check('sync bn pair', f'{what} rank {k} {tag} dy', o['dy' + tag.lower()], v, a)
    assert W == len(local)


# ------------------------------------------------------------------ generic path (VAN / ConvFormer)
@pytest.mark.parametrize('c,parts', [(96, (2000, 1136)), (320, (700, 300, 568))])
@pytest.mark.parametrize('x_f32,g_f32,dx_f32,with_dres', [(False, False, False, False), (True, True, True, True),
                                                          (True, False, True, False), (False, True, False, True)])
def test_generic_sync_bn_conforms(c, parts, x_f32, g_f32, dx_f32, with_dres):
    rows = sum(parts)
    W = len(parts)
    x, gamma, beta, rm0, rv0 = _case(rows, c, 400 + c, f32=x_f32)
    g = randn(rows, c, seed=410 + c)
    g = g if g_f32 else g.to(torch.bfloat16)
    dres = randn(rows, c, seed=420 + c) if with_dres else None
    xs, gs = _split(x, parts), _split(g, parts)
    dress = _split(dres, parts) if with_dres else [None] * W
    stats = []
    for xk in xs:
        ops.partial_ws(x.device, 2 * c).fill_(NAN)
        part, prow = ops.bn_stats_generic(xk)
        stats.append(_fold(part, xk.shape[0], c, prow))
    total = _allreduce(stats)
    o = _finalize_folded(total, c, gamma, beta, rm0, rv0)
    what = f'generic sync bn c {c} parts {parts} x {"f32" if x_f32 else "bf16"} g {"f32" if g_f32 else "bf16"}'
    _check_finalize('generic sync bn stats', what, x, gamma, beta, rm0, rv0, o,
                    max(_generic_stats_depth(r, c) for r in parts) + W - 1)
    local = [ops.bn_bwd_generic_reduce(xk, gk, o['saved']) for xk, gk in zip(xs, gs)]
    gsum = _allreduce(local)
    mean, rstd = o['saved'][0].double(), o['saved'][1].double()
    k1 = gamma.double() * rstd
    m0, m1 = gsum[:c].double() / rows, gsum[c:].double() / rows
    for k, (xk, gk, rk) in enumerate(zip(xs, gs, dress)):
        dg, db = nan(c), nan(c)
        dx = ops.bn_bwd_generic_apply(xk, gk, o['saved'], gamma, gsum, dg, db, dres=rk, dx_f32=dx_f32,
                                      local_sums=local[k], count=ops.bn_sync_count(total, c))
        g64 = gk.double()
        xh = (xk.double() - mean) * rstd
        t1 = g64 * xh
        depth = _generic_bwd_depth(parts[k], c)
        check('generic sync bn backward', f'{what} rank {k} dbeta (local)', db, g64.sum(0),
              (depth + 1) * U * g64.abs().sum(0))
        check('generic sync bn backward', f'{what} rank {k} dgamma (local)', dg, t1.sum(0),
              (depth + 3) * U * t1.abs().sum(0))
        v = k1 * (g64 - m0 - xh * m1)
        a = k1.abs() * 8 * U * (g64.abs() + m0.abs() + (xh * m1).abs()) + 2 * U * v.abs()
        if rk is not None:
            v = v + rk.double()
            a = rnd(v, a)
        check('generic sync bn backward', f'{what} rank {k} dx', dx, v, a)


# ------------------------------------------------------------------ invariants: one rank is the unsynchronized path
def _finalize_pair(partials, prow, rows, c, seed):
    gamma, beta = randn(c, seed=seed) * 0.5 + 1, randn(c, seed=seed + 1) * 0.5
    rm0, rv0 = randn(c, seed=seed + 2) * 0.1, rand(c, seed=seed + 3) + 0.5
    a = {'ss': nan(2, c), 'saved': nan(2, c), 'rm': rm0.clone(), 'rv': rv0.clone()}
    ops.bn_finalize(partials, gamma, beta, a['rm'], a['rv'], a['ss'], a['saved'], rows, EPS, MOM, partial_rows=prow)
    stats = ops.bn_stats_fold(partials, rows, c, partial_rows=prow)
    b = _finalize_folded(stats, c, gamma, beta, rm0, rv0)
    return a, b, stats, gamma


@pytest.mark.parametrize('source', ['bn_stats', 'gemm_epilogue', 'generic_bf16', 'generic_f32'])
@pytest.mark.parametrize('c', [64, 256])
def test_one_rank_fold_finalize_is_bn_finalize(source, c):
    rows = 6272
    if source == 'gemm_epilogue':
        k = 128
        xin = randn(rows, k, seed=900).to(torch.bfloat16)
        w = (randn(c, k, seed=901) * 0.1).to(torch.bfloat16)
        partials = ops.partial_ws(xin.device, 2 * c)
        ops.linear_fwd(xin, w, stats=partials)
        prow = ops.gemm_stats_rows(rows, c)
    elif source == 'bn_stats':
        partials, prow = ops.bn_stats(randn(rows, c, seed=902).to(torch.bfloat16)), 0
    else:
        x = randn(rows, c, seed=903) * 1.5 + 0.3
        partials, prow = ops.bn_stats_generic(x if source == 'generic_f32' else x.to(torch.bfloat16))
    a, b, _, _ = _finalize_pair(partials, prow, rows, c, 910)
    for key in a:
        exact('one-rank fold + finalize', f'{source} c {c}: {key}', b[key], a[key])


@pytest.mark.parametrize('c', [64, 512])
def test_one_rank_sync_backward_is_plain_backward(c):
    rows = 5000
    y = randn(rows, c, seed=920).to(torch.bfloat16)
    yb = randn(rows, c, seed=921).to(torch.bfloat16)
    dout = randn(rows, c, seed=922).to(torch.bfloat16)
    fa, _, stats, gamma = _finalize_pair(ops.bn_stats(y), 0, rows, c, 930)
    fb, _, _, gamma_b = _finalize_pair(ops.bn_stats(yb), 0, rows, c, 940)
    count = ops.bn_sync_count(stats, c)
    bits = ops.mask_bits_like(y)
    ops.bn_apply(y, fa['ss'], torch.empty_like(y), 1, mask_bits=bits)
    sums = nan(2, c)
    ops.bn_bwd_reduce(dout, None, y, fa['saved'], sums, 1, bits=bits)
    outs = []
    for sync in (False, True):
        o = [torch.full_like(y, NAN), torch.full_like(y, NAN), nan(c), nan(c)]
        kw = {'local_sums': sums.clone(), 'count': count} if sync else {}
        ops.bn_bwd_apply(dout, None, y, fa['saved'], gamma, sums, *o, 1, bits=bits, **kw)
        outs.append(o)
    for name, p, q in zip(('dy', 'dres', 'dgamma', 'dbeta'), *outs):
        exact('one-rank sync backward', f'apply c {c}: {name}', q, p)
    sums4 = nan(4, c)
    ops.bn_bwd_reduce2(dout, bits, y, yb, fa['saved'], fb['saved'], sums4)
    outs = []
    for sync in (False, True):
        o = [torch.full_like(y, NAN), torch.full_like(y, NAN)] + [nan(c) for _ in range(4)]
        kw = {'local_sums': sums4.clone(), 'count': count} if sync else {}
        ops.bn_bwd_apply2(dout, bits, y, yb, fa['saved'], fb['saved'], gamma, gamma_b, sums4, *o, **kw)
        outs.append(o)
    for name, p, q in zip(('dya', 'dyb', 'dga', 'dba', 'dgb', 'dbb'), *outs):
        exact('one-rank sync backward', f'apply2 c {c}: {name}', q, p)


@pytest.mark.parametrize('x_f32,g_f32,dx_f32,with_dres', [(False, False, False, False), (True, True, True, True),
                                                          (True, False, False, True)])
def test_split_generic_backward_is_bn_bwd_generic(x_f32, g_f32, dx_f32, with_dres):
    rows, c = 6272, 320
    x = randn(rows, c, seed=950) * 1.5 + 0.3
    x = x if x_f32 else x.to(torch.bfloat16)
    g = randn(rows, c, seed=951)
    g = g if g_f32 else g.to(torch.bfloat16)
    dres = randn(rows, c, seed=952) if with_dres else None
    part, prow = ops.bn_stats_generic(x)
    fo, _, stats, gamma = _finalize_pair(part, prow, rows, c, 960)
    dg0, db0 = nan(c), nan(c)
    dx0 = ops.bn_bwd_generic(x, g, fo['saved'], gamma, dg0, db0, dres=dres, dx_f32=dx_f32)
    sums = ops.bn_bwd_generic_reduce(x, g, fo['saved'])
    for kw in ({}, {'local_sums': sums.clone(), 'count': ops.bn_sync_count(stats, c)}):
        dg, db = nan(c), nan(c)
        dx = ops.bn_bwd_generic_apply(x, g, fo['saved'], gamma, sums, dg, db, dres=dres, dx_f32=dx_f32, **kw)
        tag = 'sync' if kw else 'split'
        exact('one-rank generic backward', f'{tag}: dx', dx, dx0)
        exact('one-rank generic backward', f'{tag}: dgamma', dg, dg0)
        exact('one-rank generic backward', f'{tag}: dbeta', db, db0)


def test_row_count_is_exact_beyond_2_24():
    """Two ranks of 2^24 + 1 and 2^24 + 2 rows (the sum, 2^25 + 3, has no fp32 representation): the summed count slots
    decode to the exact global count, and finalize uses it (mean = sum * (1 / (float)n), unbiased factor n / (n - 1))."""
    c = 64
    n0, n1 = 2 ** 24 + 1, 2 ** 24 + 2
    sums = [torch.stack([randn(c, seed=970 + k) * 1e3, rand(c, seed=975 + k) * 1e9]).reshape(1, 2 * c).contiguous()
            for k in range(2)]
    total = _allreduce([ops.bn_stats_fold(s, n, c, partial_rows=1) for s, n in zip(sums, (n0, n1))])
    n = n0 + n1
    assert int(total[2 * c].item()) * 4096 + int(total[2 * c + 1].item()) == n
    gamma, beta = torch.ones(c, device='cuda'), torch.zeros(c, device='cuda')
    o = _finalize_folded(total, c, gamma, beta, torch.zeros(c, device='cuda'), torch.ones(c, device='cuda'))
    want = nan(2, c)
    ref = {'ss': nan(2, c), 'saved': want, 'rm': torch.zeros(c, device='cuda'), 'rv': torch.ones(c, device='cuda')}
    ops.bn_finalize(total[:2 * c].contiguous(), gamma, beta, ref['rm'], ref['rv'], ref['ss'], ref['saved'], n, EPS, MOM,
                    partial_rows=1)
    for key in ('ss', 'saved', 'rm', 'rv'):
        same(f'count beyond 2^24: {key}', o[key], ref[key])
