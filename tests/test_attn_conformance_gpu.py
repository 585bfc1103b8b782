"""Conformance of the wgmma attention family (csrc/attn_sm90.cuh through saicv_attn_fwd / saicv_attn_bwd) against float64
interval references, and its bit-identity invariants.

Every reference is computed on the GPU in float64 from the same bf16 operands, batched over (b, h).  Each quantisation
step the kernel takes is mirrored as an interval, and every output element must lie in the bf16 rounding of its interval
(no fraction of misses is allowed).  Notation, per (b, h): sigma is the fp32 scale, c = fl32(sigma * fl32(log2 e)) as
capi_attn.cu forms scale_log2, s = q k^T exact, e_s = 2^-16 |q| |k|^T the fp32 accumulation allowance of the m64n64 k16
wgmma chain (the GEMM suite's rule), U = 2^-24 one fp32 rounding, and 2^-21 the relative error allowed for ex2.approx and
__fdividef (the PTX ISA documents a few ulps).  Dead keys are the masked ones and those past Lk.

Forward.  Key block J covers keys [64J, 64J + 64); M_J is the running maximum of s over live keys up to block J and M
the row's final one; e_max is the largest e_s of a live key in the row.  The kernel forms P relative to its own running
maximum (of the rounded scores, within e_max of M_J) and rounds it to bf16 there, before any later rescale:
  * exponent (s - M_J) c, off by at most dx = c (e_s + e_max) + 2^-23 c (|s| + |M_J|) (the fmaf and the rounding of
    M_J c); the fp32 weight lies in [2^(x - dx) (1 - 2^-21), 2^(x + dx) (1 + 2^-21)], with a lower end of 0 below 2^-125
    (ex2.approx.ftz flushes).  With dropout: times keep * fl32(1 / (1 - fl32(p))), one more U, kept or 0;
  * the bf16 weight w lies in [rne(lo), rne(hi)];
  * the later rescales multiply by 2^((M_J - M) c) up to kappa = 2^delta (1 + nkb (2^-21 + U)) - 1, where
    delta = 2 c e_max + 2^-23 c (M - M_J + 2 e_max) (the telescoped corr exponents and their roundings);
  * numerator centre sum mid(w) Pi v, radius sum (half(w) + kappa |w| + 2^-16 (1 + kappa) |w|) Pi |v| + 2^-22 |centre|;
  * denominator l = sum over live keys of 2^((s - M) c), **undropped**; relative radius max over keys of
    (2^dx (1 + 2^-21) - 1) + max kappa + (2 nkb + 20) U + Lk 2^-126 / l;
  * O = numerator / l, then __fdividef and the product: (2^-21 + U) relative.  The stored bf16 O must lie in
    [rne(lo), rne(hi)].  lse (log2 domain) must lie within c e_max + 2 U |M c| + eps_l / ln 2 + 2^-22 |log2 l| +
    2 U |lse| of M c + log2 l.  A row without live keys must give O = 0 and lse = -inf exactly.
Backward, at the saved state (the kernel's own bf16 O and fp32 lse, so it is checked independently of the forward):
  * p = 2^(s c - lse), exponent off by c e_s + U |s c - lse|, plus 2^-21, lower end 0 below 2^-125;
  * dP = dO v^T within 2^-16 |dO| |v|^T; D = sum dO O within 2^-20 sum |dO O| (attn_delta_kernel: exact bf16 products,
    at most 16 fp32 adds); with dropout dP' = keep dP fl32(1 / (1 - p)) plus U;
  * dS = p (dP' - D) with the propagated radius, one U for the subtraction and one for the product; its bf16 value lies
    in [rne(lo), rne(hi)], and is exactly 0 for a dead key;
  * dQ = sigma sum_t dS k and dK = sigma sum_i dS^T q (first dk_cols columns): centre mid(dS) @ k, radius
    half(dS) @ |k| + 2^-16 |dS| @ |k| + 2^-22 |centre|, then one U for the sigma product;
  * dV = sum_i P~^T dO with P~ = rne(keep p fl32(1 / (1 - p))) as an interval, radius as for dQ.
Dead keys therefore get exactly 0 in dK and dV, and the queries of a batch element without live keys exactly 0 in dQ.

Each check prints max |out - centre| / S (S the absolute sum of the check: sum |w| Pi |v| / l for O, the |dS| or |P~|
products for the gradients) and the largest fraction of the allowance any element used; run with -s to see them.
Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit: lse uses at most 0.4 % of its allowance, O at most 82 %,
dQ, dK and dV up to 99.6 %.  The bf16 flips of P and dS dominate: when only one P~ or dS of a row lies within its own
error of a rounding boundary, the kernel's choice moves the output by that value's whole half-width, which is then
nearly all of the allowance.  The continuous terms (e_s, ex2, the corr chain) are small next to one bf16 step.  The
file runs in about 11 s.

Invariants (compared as raw bits):
  * item independence: each (b, h) of a launch with more work items than resident CTAs, an odd number of query and key
    blocks and a key mask equals the same (b, h) launched alone (fwd O and lse, bwd dQ, dK and dV; the dropout hash row
    depends on b H + h, so dropout is left out).  Unreset m, l or O, or a ring phase that reads stale K / V, fail it;
  * layout independence: contiguous [B, H, L, D], packed [B, L, 3, H, D] views and views with slack between rows;
  * owned writes: output storage with slack rows and columns is filled with a NaN sentinel; after the launches
    everything outside the O, dQ, dK and dV views, and dK's columns from dk_cols on, still holds it.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conformance import M32, U, check, drop_scale, dropout_hash, dropout_keep, dropout_threshold, rne_bf16, same

from simpleaicv_pytorch_training_examples_b200 import _lib, ops

APPROX = 2.0 ** -21     # ex2.approx, __fdividef, relative
ACC = 2.0 ** -16        # wgmma fp32 accumulation, relative to the absolute product sum
TINY = 2.0 ** -125      # below this an ex2.approx.ftz result may be flushed to zero
WIDTHS = [(32, 32), (48, 32), (64, 64), (80, 80), (96, 64), (112, 64), (112, 80), (128, 80), (192, 64), (208, 80)]
DROP_WIDTHS = [(32, 32), (48, 32), (64, 64)]
SENTINEL = 0x7FA5       # a bf16 NaN the kernels never produce


# ------------------------------------------------------------------ the counter hash copy (conformance.py) against the C ABI
def _seed_hashing_element0_to(h):
    """A seed (high word 0) whose hash of element (0, 0) is h: the finaliser is a bijection, invert it."""
    x = h ^ (h >> 16)
    x = x * pow(0x846CA68B, -1, 1 << 32) & M32
    x ^= (x >> 15) ^ (x >> 30)
    x = x * pow(0x7FEB352D, -1, 1 << 32) & M32
    x ^= x >> 16
    return x * pow(0x9E3779B1, -1, 1 << 32) & M32


# p = 0.1: the double threshold is 429496729, the fp32 one 429496736.  This seed puts element 0 between them, so a copy
# of the hash that thresholds the double p keeps an element the kernels drop.
SEED_BETWEEN = _seed_hashing_element0_to(int(0.1 * 4294967296.0))


def test_dropout_hash_copy_and_threshold_cpu():
    """The torch copy of the hash against plain 32-bit integer arithmetic, and the threshold from the fp32 p."""
    def ref(seed, a, b):
        x = ((a + (seed & M32)) & M32) * 0x9E3779B1 & M32
        x ^= ((b + (seed >> 32)) & M32) * 0x85EBCA77 & M32
        x ^= x >> 16
        x = x * 0x7FEB352D & M32
        x ^= x >> 15
        x = x * 0x846CA68B & M32
        return x ^ (x >> 16)

    g = torch.Generator().manual_seed(0)
    a = torch.randint(0, 1 << 32, (2000,), generator=g, dtype=torch.int64)
    b = torch.randint(0, 1 << 32, (2000,), generator=g, dtype=torch.int64)
    for seed in (0, 0x0123456789ABCDEF, 0xFFFFFFFFFFFFFF00):
        got = dropout_hash(seed, a, b).tolist()
        assert got == [ref(seed, x, y) for x, y in zip(a.tolist(), b.tolist())]
    assert dropout_threshold(0.1) - int(0.1 * 4294967296.0) == 7
    assert dropout_threshold(0.2) - int(0.2 * 4294967296.0) == 13
    assert dropout_threshold(0.5) == 1 << 31 and dropout_threshold(0.0) == 0
    zero = torch.zeros(1, dtype=torch.int64)
    assert dropout_hash(SEED_BETWEEN, zero, zero).item() == int(0.1 * 2 ** 32)
    assert not dropout_keep(SEED_BETWEEN, zero, zero, 0.1).item()
    assert drop_scale(0.1) == float(np.float32(1) / np.float32(0.9))


@pytest.mark.gpu
@pytest.mark.parametrize('p,seed', [(0.1, 0x0123456789ABCDEF), (0.5, 0xFFFFFFFFFFFFFF00), (0.1, SEED_BETWEEN)])
def test_dropout_hash_copy_matches_device(p, seed):
    """ops.dropout on ones keeps exactly the hash(seed, i mod 2^32, i >> 32) mask (capi_detr.cu's indexing), which pins
    the torch copy the attention references use."""
    n = 1 << 16
    got = ops.dropout(torch.ones(n, device='cuda', dtype=torch.bfloat16), p, seed) != 0
    i = torch.arange(n, device='cuda', dtype=torch.int64)
    want = dropout_keep(seed, i & M32, i >> 32, p)
    assert torch.equal(got, want), f'{int((got != want).sum())} of {n} keep decisions differ'


# ------------------------------------------------------------------ operands, masks
def _c(sigma):
    return float(np.float32(np.float32(sigma) * np.float32(1.4426950408889634)))


def _operands(B, H, Lq, Lk, dqk, dv, regime='random', seed=0):
    """q, k, v bf16 [B, H, L, D] laid out as the runtimes lay them out, and the softmax scale.  Plain widths use
    sigma = hd^-1/2.  DETR (48, 32): pre-scaled q, q column 32 = 1, the 0/1 key bias in k column 32, zeros after.  SAM
    (dqk > dv): pre-scaled q, rel-pos values in q and one-hot (kh, kw) in k on an S x S grid (capi_sam.cu), zeros after."""
    g = torch.Generator(device='cuda').manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, device='cuda', generator=g)

    hd, nb = dv, dqk - dv
    q, k = torch.zeros(B, H, Lq, dqk, device='cuda'), torch.zeros(B, H, Lk, dqk, device='cuda')
    if nb == 0:
        sigma = hd ** -0.5
        q, k = rn(B, H, Lq, dqk), rn(B, H, Lk, dqk)
    elif (dqk, dv) == (48, 32):
        sigma = 1.0
        q[..., :hd], k[..., :hd] = rn(B, H, Lq, hd) * hd ** -0.5, rn(B, H, Lk, hd)
        q[..., hd] = 1.0
        k[..., hd] = torch.randint(0, 2, (B, 1, Lk), device='cuda', generator=g).float()
    else:
        sigma = 1.0
        S = 64 if nb >= 128 else 14
        q[..., :hd], k[..., :hd] = rn(B, H, Lq, hd) * hd ** -0.5, rn(B, H, Lk, hd)
        q[..., hd:hd + 2 * S] = rn(B, H, Lq, 2 * S)
        pos = torch.arange(Lk, device='cuda')
        k[:, :, pos, hd + (pos // S) % S] = 1.0
        k[:, :, pos, hd + S + pos % S] = 1.0
    v = rn(B, H, Lk, dv)
    c = _c(sigma)
    blk = (torch.arange(Lk, device='cuda') // 64).float()
    if regime == 'rising':        # the row maximum rises by about 4 (log2 units) in every key block
        q[..., 0] = 2.0
        k[..., 0] = blk * (2.0 / c)
    elif regime == 'falling':     # maximum in block 0, the tail 80 log2 units lower per block: below 2^-126 from block 2
        q[..., 0] = 2.0
        k[..., 0] = -blk * (40.0 / c)
    elif regime == 'peaked':      # plain widths: query i has one key at p ~ 1, the rest below 2^-30
        t = (torch.arange(Lq, device='cuda') * 7) % Lk
        q = 8.0 * k.bfloat16().float()[:, :, t]
    elif regime != 'random':
        raise ValueError(regime)
    return q.bfloat16(), k.bfloat16(), v.bfloat16(), sigma


def _mask(kind, B, Lk, seed=0):
    """dead bool [B, Lk] (None without a mask) and the packed bits.  Bits of keys >= Lk are set (the kernels must
    ignore them).  'holes': random keys at odd and even positions; 'block': the first key and the whole second block;
    'prefix': valid prefixes ending on block boundaries, the last batch element fully masked; 'wide': holes with four
    more mask words than the minimum."""
    if kind is None:
        return None, None
    g = torch.Generator(device='cuda').manual_seed(seed + 99)
    dead = torch.zeros(B, Lk, dtype=torch.bool, device='cuda')
    if kind in ('holes', 'wide'):
        dead = torch.rand(B, Lk, device='cuda', generator=g) < 0.3
    elif kind == 'block':
        dead[:, 0] = True
        dead[:, 64:128] = True
        dead[:, 131] = dead[:, 140] = True
    elif kind == 'prefix':
        for b in range(B):
            dead[b, min(64 * (b % 2 + 1), Lk):] = True
        dead[-1] = True
    else:
        raise ValueError(kind)
    words = (Lk + 127) // 128 * 4 + (4 if kind == 'wide' else 0)
    full = torch.ones(B, words * 32, dtype=torch.bool, device='cuda')
    full[:, :Lk] = dead
    return dead, ops.pack_key_mask(full, words * 32)


def _keep_mask(B, H, Lq, Lk, p, seed):
    """keep [B, H, Lq, Lk] of the attention kernels: hash row (b H + h) Lq + q, column key."""
    rows = torch.arange(B * H * Lq, device='cuda', dtype=torch.int64).view(B, H, Lq, 1)
    cols = torch.arange(Lk, device='cuda', dtype=torch.int64).view(1, 1, 1, Lk)
    return dropout_keep(seed, rows, cols, p)


def _live(dead, shape):
    if dead is None:
        return torch.ones(shape, dtype=torch.bool, device='cuda')
    return (~dead)[:, None, None, :].expand(shape)


# ------------------------------------------------------------------ float64 interval references
def _scores(q, k):
    qd, kd = q.double(), k.double()
    return qd @ kd.transpose(-1, -2), ACC * (qd.abs() @ kd.abs().transpose(-1, -2))


def _fwd_ref(q, k, v, sigma, dead, keep, dscale):
    """Centre and allowance of O, its absolute sum, centre and allowance of lse, and which rows have live keys."""
    c = _c(sigma)
    s, es = _scores(q, k)
    B, H, Lq, Lk = s.shape
    nkb = (Lk + 63) // 64
    live = _live(dead, s.shape)
    ninf = torch.tensor(float('-inf'), dtype=torch.float64, device='cuda')
    bm = F.pad(torch.where(live, s, ninf), (0, nkb * 64 - Lk), value=float('-inf')).view(B, H, Lq, nkb, 64).amax(-1)
    MJ = bm.cummax(-1).values
    rowlive = MJ[..., -1:] > float('-inf')
    Mf = torch.where(rowlive, MJ[..., -1:], 0.0)
    Mt = torch.where(live, MJ.repeat_interleave(64, -1)[..., :Lk], 0.0)
    emax = torch.where(live, es, 0.0).amax(-1, keepdim=True)
    x = torch.where(live, (s - Mt) * c, ninf)
    dx = torch.where(live, c * (es + emax) + 2.0 ** -23 * c * (s.abs() + Mt.abs()), 0.0)
    plo = torch.exp2(x - dx) * (1 - APPROX)
    phi = torch.exp2(x + dx) * (1 + APPROX)
    plo = torch.where(phi < TINY, 0.0, plo)
    pi = torch.where(live, torch.exp2((Mt - Mf) * c), 0.0)
    delta = 2 * c * emax + 2.0 ** -23 * c * (Mf - Mt + 2 * emax)
    kap = torch.where(live, torch.exp2(delta) * (1 + nkb * (APPROX + U)) - 1, 0.0)
    l = torch.where(live, torch.exp2((s - Mf) * c), 0.0).sum(-1, keepdim=True)
    l1 = torch.where(rowlive, l, 1.0)
    eps = (torch.where(live, torch.exp2(dx) * (1 + APPROX) - 1, 0.0).amax(-1, keepdim=True) + kap.amax(-1, keepdim=True)
           + (2 * nkb + 20) * U + Lk * 2.0 ** -126 / l1)
    del s, es, x, dx, Mt
    if keep is not None:
        plo = torch.where(keep, plo * dscale * (1 - U), 0.0)
        phi = torch.where(keep, phi * dscale * (1 + U) + 2.0 ** -149, 0.0)
    wlo, whi = rne_bf16(plo), rne_bf16(phi)
    del plo, phi
    vd = v.double()
    num = ((wlo + whi) / 2 * pi) @ vd
    rnum = (((whi - wlo) / 2 + kap * whi + ACC * (1 + kap) * whi) * pi) @ vd.abs() + 2.0 ** -22 * num.abs()
    s_abs = (whi * pi) @ vd.abs() / l1
    o = num / l1
    a = rnum / l1 / (1 - eps) + o.abs() * eps / (1 - eps)
    a = a + (o.abs() + a) * (APPROX + U)
    lse = Mf[..., 0] * c + torch.log2(l1[..., 0])
    lse_a = (c * emax + 2 * U * (Mf * c).abs() + eps / math.log(2) / (1 - eps) + 2.0 ** -22 * torch.log2(l1).abs())[..., 0]
    lse_a = lse_a + 2 * U * lse.abs()
    return o, a, s_abs, lse, lse_a, rowlive[..., 0]


def _mm_interval(lo, hi, b, scale=1.0):
    """Centre, allowance and absolute sum of scale * (X @ b) for X in the elementwise interval [lo, hi] (bf16 values)
    reduced by wgmma (2^-16 of the absolute sum), then one fp32 product with the scale."""
    bd = b.double()
    mag = torch.maximum(lo.abs(), hi.abs()) @ bd.abs()
    centre = ((lo + hi) / 2) @ bd
    rad = ((hi - lo) / 2) @ bd.abs() + ACC * mag + 2.0 ** -22 * centre.abs()
    v, a = scale * centre, scale * rad
    return v, a + U * (v.abs() + a), scale * mag


def _bwd_ref(q, k, v, o, lse, do, sigma, dead, keep, dscale):
    """(centre, allowance, absolute sum) of dQ, dK and dV at the kernel's saved state (its bf16 O and fp32 lse)."""
    c, sg = _c(sigma), float(np.float32(sigma))
    s, es = _scores(q, k)
    L = lse.double()[..., None]
    live = _live(dead, s.shape) & torch.isfinite(L)
    ninf = torch.tensor(float('-inf'), dtype=torch.float64, device='cuda')
    y = torch.where(live, s * c - torch.where(live, L, 0.0), ninf)
    dy = torch.where(live, c * es + U * y.abs(), 0.0)
    del s, es
    pc = torch.exp2(y)
    plo = torch.exp2(y - dy) * (1 - APPROX)
    phi = torch.exp2(y + dy) * (1 + APPROX)
    plo = torch.where(phi < TINY, 0.0, plo)
    del y, dy
    dod, vd = do.double(), v.double()
    dp = dod @ vd.transpose(-1, -2)
    edp = ACC * (dod.abs() @ vd.abs().transpose(-1, -2))
    prod = dod * o.double()
    D, eD = prod.sum(-1, keepdim=True), 2.0 ** -20 * prod.abs().sum(-1, keepdim=True)
    if keep is not None:
        kf = keep.double()
        rdp = kf * (edp * dscale + U * (dp.abs() + edp) * dscale)
        dp = kf * dp * dscale
    else:
        rdp = edp
    del edp
    yc = dp - D
    ry = rdp + eD
    ry = ry + U * (yc.abs() + ry)
    del dp, rdp
    ds = pc * yc
    rds = torch.maximum(phi - pc, pc - plo) * (yc.abs() + ry) + pc * ry
    rds = rds + U * (ds.abs() + rds) + 2.0 ** -149
    del yc, ry
    dslo = torch.where(live, rne_bf16(ds - rds), 0.0)
    dshi = torch.where(live, rne_bf16(ds + rds), 0.0)
    del ds, rds
    dq = _mm_interval(dslo, dshi, k, sg)
    dk = _mm_interval(dslo.transpose(-1, -2), dshi.transpose(-1, -2), q, sg)
    del dslo, dshi
    if keep is not None:
        plo = torch.where(keep, plo * dscale * (1 - U), 0.0)
        phi = torch.where(keep, phi * dscale * (1 + U) + 2.0 ** -149, 0.0)
    ptlo = torch.where(live, rne_bf16(plo), 0.0).transpose(-1, -2)
    pthi = torch.where(live, rne_bf16(phi), 0.0).transpose(-1, -2)
    del plo, phi, pc
    return dq, dk, _mm_interval(ptlo, pthi, do)


# ------------------------------------------------------------------ conformance cases
def _dk_cols(dqk, dv):
    return 32 if (dqk, dv) == (48, 32) else dqk   # DETR stores dK's head columns only


def _run(B, H, Lq, Lk, dqk, dv, regime='random', mask=None, p=0.0, seed=0xFFFFFFFFFFFFFF00, tag=''):
    q, k, v, sigma = _operands(B, H, Lq, Lk, dqk, dv, regime, seed=B * 7 + Lq + 3 * Lk + dqk)
    dead, bits = _mask(mask, B, Lk, seed=Lq + Lk)
    keep = _keep_mask(B, H, Lq, Lk, p, seed) if p > 0 else None
    dscale = drop_scale(p) if p > 0 else 1.0
    what = f'{tag}B{B} H{H} Lq{Lq} Lk{Lk} ({dqk},{dv}) {regime} mask={mask} p={p}'
    out, lse = ops.attn_fwd(q, k, v, sigma, mask_bits=bits, dropout_p=p, dropout_seed=seed)
    oc, oa, os_, lc, la, rowlive = _fwd_ref(q, k, v, sigma, dead, keep, dscale)
    check(None, f'O {what}', out, oc, oa, os_)
    assert torch.equal(lse[~rowlive], torch.full_like(lse[~rowlive], float('-inf'))), f'lse {what}: rows without keys'
    if rowlive.any():
        check(None, f'lse {what}', lse[rowlive], lc[rowlive], la[rowlive], torch.ones_like(la[rowlive]))
    del oc, oa, os_, lc, la
    g = torch.Generator(device='cuda').manual_seed(Lq * 31 + Lk)
    do = torch.randn(B, Lq, H, dv, device='cuda', generator=g).bfloat16().permute(0, 2, 1, 3)   # the layout of out
    dq, dk, dvv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    dkc = _dk_cols(dqk, dv)
    ops.attn_bwd(q, k, v, out, lse, do, sigma, dq, dk, dvv, dk_cols=dkc, mask_bits=bits, dropout_p=p, dropout_seed=seed)
    (qc, qa, qs), (kc, ka, ks), (vc, va, vs) = _bwd_ref(q, k, v, out, lse, do, sigma, dead, keep, dscale)
    check(None, f'dQ {what}', dq, qc, qa, qs)
    check(None, f'dK {what}', dk[..., :dkc], kc[..., :dkc], ka[..., :dkc], ks[..., :dkc])
    check(None, f'dV {what}', dvv, vc, va, vs)


CASES = []
for _i, (_q, _v) in enumerate(WIDTHS):
    CASES += [(2, 3, (130, 196, 197)[_i % 3], (130, 196, 197)[_i % 3], _q, _v, 'random', None, 0.0),
              (2, 2, 70, 250, _q, _v, 'random', 'holes', 0.0),        # cross attention, Lq < Lk
              (2, 2, 250, 100, _q, _v, 'random', 'prefix', 0.0)]      # Lq > Lk, a fully masked batch element
CASES += [(1, 2, 300, 300, dq_, dv_, rg, None, 0.0) for dq_, dv_ in ((64, 64), (208, 80)) for rg in ('rising', 'falling')]
CASES += [(2, 2, 200, 200, 64, 64, 'peaked', None, 0.0),
          (2, 2, 200, 330, 64, 64, 'random', 'block', 0.0),
          (3, 2, 150, 260, 32, 32, 'random', 'wide', 0.0),
          (2, 2, 150, 300, 208, 80, 'rising', 'holes', 0.0),
          (1, 1, 4096, 4096, 192, 64, 'random', None, 0.0),          # SAM global attention: 64 key blocks
          (1, 1, 4096, 4096, 208, 80, 'random', None, 0.0),
          (6, 16, 150, 150, 64, 64, 'random', 'holes', 0.0),         # 288 items on 264 resident CTAs, 3 x 3 blocks
          (4, 12, 150, 150, 208, 80, 'random', 'holes', 0.0)]        # 144 items on 132 resident CTAs
CASES += [(2, 4, 130, 150, dq_, dv_, 'random', m, p) for dq_, dv_ in DROP_WIDTHS for p in (0.1, 0.5) for m in (None, 'holes')]
CASES += [(2, 2, 100, 130, 32, 32, 'random', 'prefix', 0.1), (2, 6, 150, 150, 64, 64, 'falling', 'block', 0.1)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,H,Lq,Lk,dqk,dv,regime,mask,p', CASES)
def test_attn_conforms(B, H, Lq, Lk, dqk, dv, regime, mask, p):
    _run(B, H, Lq, Lk, dqk, dv, regime, mask, p)


LENGTHS = [1, 2, 63, 64, 65, 127, 128, 129]


@pytest.mark.gpu
@pytest.mark.parametrize('dqk,dv', [(64, 64), (112, 80)])
def test_attn_lengths_conform(dqk, dv):
    """Every (Lq, Lk) pair around one and two 64-row / 64-key blocks."""
    for lq in LENGTHS:
        for lk in LENGTHS:
            _run(1, 2, lq, lk, dqk, dv, mask='holes' if lk > 1 else None, tag='lengths ')


# ------------------------------------------------------------------ bit-identity invariants
@pytest.mark.gpu
@pytest.mark.parametrize('B,H,L,dqk,dv', [(6, 16, 150, 64, 64), (4, 12, 150, 208, 80)])
def test_attn_items_are_independent(B, H, L, dqk, dv):
    """Each (b, h) of a launch with more items than resident CTAs equals the same (b, h) launched alone."""
    q, k, v, sigma = _operands(B, H, L, L, dqk, dv, seed=5)
    _, bits = _mask('holes', B, L, seed=5)
    do = torch.randn(B, L, H, dv, device='cuda', generator=torch.Generator(device='cuda').manual_seed(6)).bfloat16().permute(0, 2, 1, 3)
    dkc = _dk_cols(dqk, dv)
    out, lse = ops.attn_fwd(q, k, v, sigma, mask_bits=bits)
    grads = [torch.empty_like(t) for t in (q, k, v)]
    ops.attn_bwd(q, k, v, out, lse, do, sigma, *grads, dk_cols=dkc, mask_bits=bits)
    out1, lse1 = torch.empty_like(out), torch.empty_like(lse)
    grads1 = [torch.empty_like(t) for t in (q, k, v)]
    for b in range(B):
        for h in range(H):
            i = (slice(b, b + 1), slice(h, h + 1))
            _, lse1[i] = ops.attn_fwd(q[i], k[i], v[i], sigma, out=out1[i], mask_bits=bits[b:b + 1])
            ops.attn_bwd(q[i], k[i], v[i], out[i], lse[i], do[i], sigma, *(t[i] for t in grads1), dk_cols=dkc,
                         mask_bits=bits[b:b + 1])
    same('O alone vs in a multi-item launch', out1, out)
    same('lse alone vs in a multi-item launch', lse1, lse)
    for name, a, b_ in zip(('dQ', 'dK', 'dV'), grads1, grads):
        if name == 'dK':
            a, b_ = a[..., :dkc], b_[..., :dkc]
        same(f'{name} alone vs in a multi-item launch', a, b_)


def _sentinel(*shape):
    return torch.full(shape, SENTINEL, device='cuda', dtype=torch.int16).view(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize('dqk,dv,dk_cols', [(64, 64, 48), (48, 32, 32), (208, 80, 64)])
def test_attn_layouts_and_owned_writes(dqk, dv, dk_cols):
    """The same data as contiguous [B, H, L, D], packed [B, L, 3, H, D] views (dqk == dv) and views with slack between
    rows give the same bits; outputs written into sentinel-filled storage with slack leave everything else untouched."""
    B, H, L = 2, 3, 150
    q, k, v, sigma = _operands(B, H, L, L, dqk, dv, seed=9)
    _, bits = _mask('holes', B, L, seed=9)
    do = torch.randn(B, H, L, dv, device='cuda', generator=torch.Generator(device='cuda').manual_seed(10)).bfloat16()

    def run(qv, kv, vv, ov, dov, gv):
        ov.copy_(_sentinel(*ov.shape))
        dov.copy_(do)
        for t in gv:
            t.copy_(_sentinel(*t.shape))
        _, lse = ops.attn_fwd(qv, kv, vv, sigma, out=ov, mask_bits=bits)
        ops.attn_bwd(qv, kv, vv, ov, lse, dov, sigma, *gv, dk_cols=dk_cols, mask_bits=bits)
        return [ov, lse, gv[0], gv[1][..., :dk_cols], gv[2]]

    names = ('O', 'lse', 'dQ', 'dK', 'dV')
    base = run(q, k, v, torch.empty(B, H, L, dv, device='cuda', dtype=torch.bfloat16), torch.empty_like(do),
               [torch.empty_like(t) for t in (q, k, v)])

    # slack: 5 spare rows, 24 spare columns (48 bytes) in every operand and output
    def slack(t, fill=None):
        st = _sentinel(*t.shape[:2], t.shape[2] + 5, t.shape[3] + 24) if fill is None else torch.zeros(
            *t.shape[:2], t.shape[2] + 5, t.shape[3] + 24, device='cuda', dtype=torch.bfloat16)
        view = st[:, :, :t.shape[2], :t.shape[3]]
        if fill is not None:
            view.copy_(fill)
        return st, view

    (_, qs), (_, ks), (_, vs) = slack(q, q), slack(k, k), slack(v, v)
    (ost, ov), (_, dov) = slack(base[0]), slack(do, do)
    gst = [slack(t) for t in (q, k, v)]
    got = run(qs, ks, vs, ov, dov, [g[1] for g in gst])
    for n, a, b in zip(names, got, base):
        same(f'{n} with slack between rows vs contiguous', a, b)
    owned = [(ost, dv), (gst[0][0], dqk), (gst[1][0], dk_cols), (gst[2][0], dv)]
    for n, (st, cols) in zip(('O', 'dQ', 'dK', 'dV'), owned):
        region = torch.zeros(st.shape, dtype=torch.bool, device='cuda')
        region[:, :, :L, :cols] = True
        bits16 = st.view(torch.int16)
        assert (bits16[~region] == SENTINEL).all(), f'{n}: {int((bits16[~region] != SENTINEL).sum())} elements outside the view were written'
        assert (bits16[region] != SENTINEL).all(), f'{n}: {int((bits16[region] == SENTINEL).sum())} owned elements were not written'

    if dqk == dv:
        qkv = torch.stack([q, k, v], 2).permute(0, 3, 2, 1, 4).contiguous()   # [B, L, 3, H, D]
        qp, kp, vp = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))
        op = torch.empty(B, L, H, dv, device='cuda', dtype=torch.bfloat16).permute(0, 2, 1, 3)
        dop = torch.empty(B, L, H, dv, device='cuda', dtype=torch.bfloat16).permute(0, 2, 1, 3)
        dqkv = torch.empty_like(qkv)
        got = run(qp, kp, vp, op, dop, [dqkv[:, :, i].permute(0, 2, 1, 3) for i in range(3)])
        for n, a, b in zip(names, got, base):
            same(f'{n} packed [B, L, 3, H, D] vs contiguous', a, b)
        assert (dqkv[:, :, 1, :, dk_cols:].contiguous().view(torch.int16) == SENTINEL).all(), 'dK columns >= dk_cols written'


@pytest.mark.gpu
@pytest.mark.parametrize('dqk,dv', DROP_WIDTHS)
def test_attn_dropout_seed_base_carries(dqk, dv):
    """A device seed base whose addition carries from the low seed word into the high one gives the same masks as the
    equivalent constant seed, forward and backward."""
    B, H, L, p = 2, 4, 150, 0.5
    q, k, v, sigma = _operands(B, H, L, L, dqk, dv, seed=12)
    _, bits = _mask('holes', B, L, seed=12)
    do = torch.randn(B, L, H, dv, device='cuda', generator=torch.Generator(device='cuda').manual_seed(13)).bfloat16().permute(0, 2, 1, 3)
    const, part, base = 0x0000123400000100, 0x00001233FFFFFF00, 0x200
    assert part + base == const and (part & M32) + base > M32
    runs = []
    for seed, sb in ((const, None), (part, torch.tensor([base], dtype=torch.int64, device='cuda'))):
        out, lse = ops.attn_fwd(q, k, v, sigma, mask_bits=bits, dropout_p=p, dropout_seed=seed, dropout_seed_base=sb)
        grads = [torch.empty_like(t) for t in (q, k, v)]
        ops.attn_bwd(q, k, v, out, lse, do, sigma, *grads, dk_cols=_dk_cols(dqk, dv), mask_bits=bits, dropout_p=p,
                     dropout_seed=seed, dropout_seed_base=sb)
        grads[1] = grads[1][..., :_dk_cols(dqk, dv)]
        runs.append([out, lse, *grads])
    for n, a, b in zip(('O', 'lse', 'dQ', 'dK', 'dV'), *runs):
        same(f'{n}: seed base carrying into the high word vs the constant seed', a, b)


# ------------------------------------------------------------------ refusals
@pytest.mark.gpu
def test_attn_refusals_launch_nothing():
    """Malformed arguments raise through _lib.call before either entry launches a kernel."""
    B, H, L = 1, 2, 200

    def operands(dqk, dv):
        q, k, v = (torch.zeros(B, H, L, d, device='cuda', dtype=torch.bfloat16) for d in (dqk, dqk, dv))
        out = torch.zeros(B, H, L, dv, device='cuda', dtype=torch.bfloat16)
        return q, k, v, out

    _, ok_bits = _mask('holes', B, L)
    short = ok_bits[:, :4].contiguous()   # 128 keys' worth, L = 200 needs 256
    fwd_bad = [((80, 80), {'dropout_p': 0.1}, 'dropout is not compiled'),
               ((72, 64), {}, 'unsupported'),
               ((64, 64), {'mask_bits': short}, 'mask_words')]
    bwd_bad = fwd_bad + [((64, 64), {'dk_cols': 24}, 'dk_cols'), ((64, 64), {'dk_cols': 80}, 'dk_cols')]
    for (dqk, dv), kw, msg in fwd_bad:
        q, k, v, out = operands(dqk, dv)
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            ops.attn_fwd(q, k, v, 0.125, out=out, **kw)
        assert _lib.launch_count() == n0, f'forward ({dqk}, {dv}) {kw}: launched before refusing'
    for (dqk, dv), kw, msg in bwd_bad:
        q, k, v, out = operands(dqk, dv)
        lse = torch.zeros(B, H, L, device='cuda')
        grads = [_sentinel(*t.shape) for t in (q, k, v)]
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            ops.attn_bwd(q, k, v, out, lse, out, 0.125, *grads, **kw)
        assert _lib.launch_count() == n0, f'backward ({dqk}, {dv}) {kw}: launched before refusing'
        assert all((t.view(torch.int16) == SENTINEL).all() for t in grads)
