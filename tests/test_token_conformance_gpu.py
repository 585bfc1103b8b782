"""Conformance of the transformer streaming and layout kernels against a float64 reference, and their bit-identity
invariants: exact-erf GELU (capi_vit.cu), token assembly and pooling (capi_vit.cu), token gather / scatter and the fill
gradient (capi_tokens.cu), dropout and per-head packing (capi_detr.cu), window partition, the positional-embedding add
and the rel-pos score columns (capi_sam.cu).

Reference.  Every check computes the exact result in float64 on the GPU from the same bf16 / fp32 values the kernel
read.  Allowances are derived from the operation, never fitted to measured errors (u = 2^-24, one fp32 rounding):
  * Data movement is bit-exact: window partition and unpartition (padding rows are +0), relpos_pack_q, the K rows and
    the T copies of relpos_gather (its one-hot key columns are bf16 1.0 and +0), relpos_shift (including the +0
    columns up to nip), heads_pack / heads_unpack at scale 1 (the extra column is rne(extra[row]) or the rounded
    constant, the rest +0), the fp32 token_gather_bwd, and the bf16 casts (dpatch, the bf16 dsrc, relpos_table), which
    must equal rne_bf16 of the fp32 value.
  * A single fp32 add is bit-exact against the float64 sum rounded once to fp32 (the sum of two floats in float64 is
    rounded once more only when it is inexact, and 53 >= 2 * 24 + 2 makes that double rounding innocuous):
    assemble_tokens, token_gather_fwd (pos by row or by pos_idx) and add_pos_embed.
  * A scale multiply then a bf16 store lands in [rne(v - u|v|), rne(v + u|v|)], v the exact value: heads_pack /
    heads_unpack with a scale, the q * scale of relpos_gather and the fmaf of relpos_dq_combine.  The scale is the
    fp32 the C entry received.
  * Sequential fp32 sums get d u sum|terms|, d counted from the kernel's loop (each add counts once, including the
    first, exact one: that covers the second-order terms):
      - assemble_tokens_bwd: d = B (the loop over the batch); with accumulate, one more rounding of prev + sum;
      - token_pool_fwd (mean): d = L - 1, then one rounding of the division;
      - token_pool_bwd: dpooled * rn(1 / (L - 1)) is two roundings; the bf16 copy multiplies by row_scale (one more)
        before its bf16 store;
      - token_fill_grad + reduce_partials: d = ceil(rows_per_slab / 8) (each of the 8 thread rows' chain) + 7 (the
        8 chains are folded sequentially, not as a tree) + nslab (the sequential fold of the slab partials), with the
        slab count mirrored from saicv_token_fill_slabs.
  * Dropout is bit-exact against the kernel's formula evaluated in float64 with one fp32 rounding per operation:
    keep(i) ? x * rn(rn(1 / (1 - p)) * row_scale[i / elems_per_scale]) : +0, then rn(+ resid), then rne to bf16 for a
    bf16 output.  keep is the counter hash of test_attn_conformance_gpu.py (_keep) on the element index, with the
    device seed base added to the seed.  Every in / out dtype pair, with and without resid, with row_scale, with
    seed_base and in place (out is x), as engine/vit.py calls it.
  * GELU on every finite bf16 input (non-finite inputs are out of scope: torch's own fp32 and fp64 GELU disagree at
    +-inf): the bf16 output lies in [rne(g - a), rne(g + a)] with a = GELU_ABS + 2u|g| (the A&S 7.1.26 erf, then
    1 - h and x * cdf round).  GELU_ABS bounds |gelu_erf - gelu|: gelu_math.cuh gives <= 2.2e-7 in float64 for
    |x| <= 12, 4e-7 here.  It is an absolute allowance: below x ~ -6, |gelu| < 1e-8 and a relative bound would be
    meaningless.  The backward, gelu_erf_grad, runs in the GEMM epilogue (test_gemm_conformance_gpu.py).
Every element must conform; no fraction may miss.  Outputs a wrapper would allocate with torch.empty are allocated
here, filled with NaN, and passed to the C entry through _lib.call, so an element that is never written fails.

Shapes are the runtime's (ViT-B/L/H at batch 256, the MAE encoder and decoder, SAM-B/H windows and rel-pos grids,
DETR queries and a 25 x 34 feature map) plus ragged ones.  Every kernel has at least one case with more items than one
sweep of its grid covers (132 * 16 blocks of 256 threads), so each grid-stride loop wraps; the fill gradient has a
case at its 128-slab cap with more than 512 rows per slab.  test_cases_wrap_every_grid_cpu checks both from the
launch mirrors.

Invariants (raw bits): two consecutive launches give identical outputs; with accumulate the output is a first call
plus the second call's value (within the allowance); each C entry's documented refusals raise and launch nothing.

Each check prints the largest fraction of its allowance an element used (0 for a bit-exact check); at the end of the
module the largest share per family is printed (run with -s).  Measured on an NVIDIA H100 80GB HBM3 at a 700 W power
limit: the rel-pos dq_combine uses 96 % of its allowance (a correctly rounded fmaf may use all of it), token_pool_bwd
85 %, assemble_tokens_bwd 56 %, GELU 34 %, token_pool_fwd 16 %, the fill gradient 3 %.  The file runs in about 11 s.
"""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name, fname):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, fname))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_gemm = _load('gemm_conformance', 'test_gemm_conformance_gpu.py')
_attn = _load('attn_conformance', 'test_attn_conformance_gpu.py')
_norm = _load('norm_conformance', 'test_norm_conformance_gpu.py')
_rne_bf16 = _gemm._rne_bf16
_keep, _drop_scale = _attn._keep, _attn._drop_scale       # _keep: the counter hash against _threshold(p)
_every_bf16, _check, _same, _nan, _randn, _rand = _norm._every_bf16, _norm._check, _norm._same, _norm._nan, _norm._randn, _norm._rand
USED = _norm.USED       # this module's own copy of the norm module: only the checks below record into it

gpu = pytest.mark.gpu

U = 2.0 ** -24          # one fp32 rounding, relative
GELU_ABS = 4e-7         # |gelu_erf - gelu| of the A&S 7.1.26 formula, plus margin
M32 = 0xFFFFFFFF
CAP = 132 * 16 * 256    # items one sweep of grid_1d covers (132 * 16 blocks of 256 threads)
FILL_SLAB_ROWS, FILL_MAX_SLABS = 512, 128
BF16, F32 = torch.bfloat16, torch.float32


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _libmod():
    from simpleaicv_pytorch_training_examples_b200 import _lib
    return _lib


def _c(name, *args):
    """Call C entry `name` on the current stream; tensors are passed as pointers, None as a null pointer."""
    ops = _ops()
    _libmod().call(name, *[ops._p(a) if isinstance(a, torch.Tensor) else a for a in args], ops._stream())


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if USED:
        print('\nlargest share of the allowance used, by family (0: bit-exact):')
        for k in sorted(USED):
            print(f'  {k:28s} {USED[k]:.3g}')


def _exact(fam, what, out, ref):
    _same(what, out, ref)
    USED.setdefault(fam, 0.0)
    print(f'{what}: bit-exact')


def _bf(t):
    """rne_bf16 of an fp32 / float64 tensor, as bf16."""
    return _rne_bf16(t.double()).to(BF16)


def _f32(x):
    return float(np.float32(x))


def _nanb(*shape):
    return _nan(*shape, dtype=BF16)


def _randb(*shape, seed=0, scale=1.0):
    return (_randn(*shape, seed=seed) * scale).to(BF16)


# ------------------------------------------------------------------ launch mirrors
def _fill_slabs(rows):
    """saicv_token_fill_slabs: slabs of the fill-gradient reduction."""
    return max(1, min(-(-rows // FILL_SLAB_ROWS), FILL_MAX_SLABS))


def _fill_depth(rows):
    nslab = _fill_slabs(rows)
    per = -(-rows // nslab)
    return -(-per // 8) + 7 + nslab


# ------------------------------------------------------------------ cases
GELU_N = [64 * 197 * 3072, 8]                                   # ViT-B/16 MLP hidden at batch 64; one vector
VIT = [(256, 196, 768), (64, 196, 1024), (32, 196, 1280), (16, 576, 1024), (3, 7, 12)]   # B, NP, C
POOL = [(256, 197, 768, 1, True), (256, 197, 768, 0, False), (512, 197, 1280, 1, False), (512, 197, 1280, 0, True),
        (3, 8, 12, 1, True), (3, 8, 12, 0, True)]              # B, L, C, mean_pool, row_scale
MAE_ENC = [(256, 768), (3, 12)]                                 # B, C: 49 of 196 patches kept, plus cls
MAE_DEC = [(256, 512), (256, 384), (512, 512), (3, 20)]         # B, C: 197 rows from 50, mask token for the rest
DROP = [  # name, n, in f32, out f32, resid, elems_per_scale (0: no row_scale), in place, p, seed, seed_base
    ('vit drop path', 256 * 197 * 768, False, True, True, 197 * 768, False, 0.1, 8 * 12 + 3, True),
    ('vit mlp hidden in place', 16 * 197 * 3072, False, False, False, 0, True, 0.1, 8 * 12 + 2, True),
    ('vit embed grad in place', 32 * 197 * 768, True, True, False, 0, True, 0.1, 0, True),
    ('detr residual', 6 * 850 * 256, True, True, True, 0, False, 0.3, (7 << 32) | 5, False),
    ('convformer cast-scale', 8 * 3136 * 64, True, False, False, 3136 * 64, False, 0.0, 0, False),
    ('bf16 to fp32 cast', 4 * 197 * 768, False, True, False, 0, False, 0.0, 0, False),
    ('ragged', 12, True, False, False, 4, False, 0.5, 3, False),
]
WIN = [(2, 64, 64, 768, 14), (1, 64, 64, 1280, 16), (2, 20, 20, 8, 14), (3, 9, 7, 768, 14), (2, 24, 40, 8, 14)]
ADDPOS = [(2, 64 * 64 * 768), (3, 7 * 9 * 12)]                  # B, per-batch elements
RELPOS = [(14, 14, 64, 25, 12), (64, 64, 80, 1, 16), (20, 20, 32, 2, 8), (5, 9, 32, 3, 2), (5, 9, 64, 3, 2),
          (5, 9, 80, 3, 2)]                                     # Sh, Sw, hd, windows, heads
RELPOS_TABLE_WRAP = (14, 14, 80, 7040)                          # Sh, Sw, hd, nip: only padding rows past 54
DETR_H, DETR_HD, DETR_DP = 8, 32, 48
HEADS = [  # B, L, ld / C, col0 / C, extra from a tensor, scale
    (24, 850, 3, 2, True, 1.0), (24, 850, 3, 0, False, DETR_HD ** -0.5), (16, 100, 2, 1, True, DETR_HD ** -0.5),
    (16, 100, 3, 1, False, 1.0), (2, 850, 2, 0, False, DETR_HD ** -0.5)]


def _wrap_items():
    """Items of each kernel's largest case, per the launches of its C entry."""
    ops = _ops()
    dqk = lambda s: ops.relpos_dqk(s[2], s[0], s[1])           # noqa: E731
    nip = lambda s: ops.relpos_nip(s[0], s[1])                 # noqa: E731
    nw = lambda h, w, ws: -(-h // ws) * -(-w // ws)            # noqa: E731
    return {
        'gelu_fwd': max(n // 8 for n in GELU_N),
        'dropout': max(n // 4 for _, n, *_ in DROP),
        'assemble_tokens': max(b * (np_ + 1) * c // 4 for b, np_, c in VIT),
        'assemble_tokens_bwd': max((np_ + 1) * c for _, np_, c in VIT),
        'token_pool_fwd': max(b * c for b, _, c, _, _ in POOL),
        'token_pool_bwd': max(b * l * c for b, l, c, _, _ in POOL),
        'token_gather_fwd / bwd': max([b * 50 * c // 4 for b, c in MAE_ENC] + [b * 197 * c // 4 for b, c in MAE_DEC]),
        'window_partition': max(b * nw(h, w, ws) * ws * ws * c // 8 for b, h, w, c, ws in WIN),
        'window_unpartition': max(b * h * w * c // 8 for b, h, w, c, _ in WIN),
        'add_pos_embed': max(b * n // 4 for b, n in ADDPOS),
        'relpos_pack_q / dq_combine': max(s[3] * s[4] * s[0] * s[1] * s[2] // 8 for s in RELPOS),
        'relpos_table': RELPOS_TABLE_WRAP[2] * RELPOS_TABLE_WRAP[3],
        'relpos_gather': max(s[3] * s[4] * s[0] * s[1] * dqk(s) // 8 for s in RELPOS),
        'relpos_shift': max(s[3] * s[4] * s[0] * s[1] * nip(s) // 8 for s in RELPOS),
        'heads_pack': max(b * DETR_H * l * DETR_DP // 8 for b, l, *_ in HEADS),
        'heads_unpack': max(b * DETR_H * l * DETR_HD // 8 for b, l, *_ in HEADS),
    }


def test_cases_wrap_every_grid_cpu():
    """Every kernel's grid-stride loop wraps in at least one case, and the fill gradient runs at its slab cap with more
    than 512 rows per slab; the Python slab mirror matches saicv_token_fill_slabs."""
    items = _wrap_items()
    short = {k: v for k, v in items.items() if v <= CAP}
    assert not short, f'cases that fit in one grid sweep of {CAP} items: {short}'
    rows = max(b * 197 for b, _ in MAE_DEC)
    nslab = _fill_slabs(rows)
    assert nslab == FILL_MAX_SLABS and -(-rows // nslab) > FILL_SLAB_ROWS
    lib = _libmod().load()
    for r in (1, 2, 511, 512, 513, 12800, 50432, 65535, 65536, 65537, 100864, 10 ** 7):
        assert lib.saicv_token_fill_slabs(r) == _fill_slabs(r), r


# ------------------------------------------------------------------ GELU
def _gelu64(x):
    return x * 0.5 * (1.0 + torch.erf(x * 0.5 ** 0.5))


@gpu
def test_gelu_on_every_bf16_input():
    """gelu_erf (forward) on every finite bf16 value."""
    u = _every_bf16(256)
    n = u.numel()
    g = _gelu64(u.double())

    def run():
        o = {'h': _nanb(*u.shape)}
        _c('saicv_gelu_fwd', u, o['h'], n)
        return o

    o = run()
    _check('gelu', 'gelu forward on every bf16 input', o['h'], g, GELU_ABS + 2 * U * g.abs())
    for k, t in run().items():
        _same(f'gelu {k} on a second launch', t, o[k])


@gpu
@pytest.mark.parametrize('n', GELU_N)
def test_gelu_streams_conform(n):
    """The MLP hidden activation of ViT-B/16 at batch 64: the grid-stride loop wraps nine times."""
    u = _randb(n, seed=2, scale=2.0)
    h = _nanb(n)
    _c('saicv_gelu_fwd', u, h, n)
    g = _gelu64(u.double())
    _check('gelu', f'gelu forward n {n}', h, g, GELU_ABS + 2 * U * g.abs())


# ------------------------------------------------------------------ dropout
def _dropout_ref(x, p, seed, resid, row_scale, eps, out_f32):
    """The kernel's formula with one fp32 rounding per operation (float64 products / sums of fp32 values, rounded)."""
    n = x.numel()
    j = torch.arange(n, device='cuda', dtype=torch.int64)
    keep = _keep(seed, j & M32, j >> 32, p)
    inv = _drop_scale(p)
    if row_scale is not None:
        sc = (inv * row_scale.double()).float().double()[j // eps]
    else:
        sc = inv
    del j
    v = (x.flatten().double() * sc).float()
    v = torch.where(keep, v, torch.zeros((), device='cuda'))
    if resid is not None:
        v = (v.double() + resid.flatten().double()).float()
    return (v if out_f32 else v.to(BF16)).view(x.shape)


@gpu
@pytest.mark.parametrize('case', DROP, ids=[d[0] for d in DROP])
def test_dropout_values_conform(case):
    """saicv_dropout values and mask, bit for bit, over the four dtype variants, resid, row_scale, seed_base, in place."""
    name, n, in_f32, out_f32, with_resid, eps, inplace, p, seed, with_base = case
    x = _randn(n, seed=10) * 3
    x = x if in_f32 else x.to(BF16)
    resid = _randn(n, seed=11) if with_resid else None
    rs = ((_rand(n // eps, seed=12) > 0.2).float() * (_rand(n // eps, seed=13) + 0.5)) if eps else None
    base = torch.tensor([123456789012345], device='cuda', dtype=torch.int64) if with_base else None
    eff_seed = (seed + (int(base.item()) if with_base else 0)) & ((1 << 64) - 1)
    ref = _dropout_ref(x, p, eff_seed, resid, rs, eps, out_f32)

    def run():
        if inplace:
            assert in_f32 == out_f32
            out = x.clone()
            src = out
        else:
            out = _nan(n, dtype=F32 if out_f32 else BF16)
            src = x
        _c('saicv_dropout', src, int(in_f32), resid, rs, eps, out, int(out_f32), n, p, seed, base)
        return out

    out = run()
    _exact('dropout', f'dropout {name} (n {n}, p {p})', out, ref)
    if p > 0 and resid is None and n > 10 ** 5:
        kept = (out != 0).double().mean().item()
        assert abs(kept - (1 - p)) < 0.01, f'{name}: kept fraction {kept}'
    _same(f'dropout {name} on a second launch', run(), out)


# ------------------------------------------------------------------ ViT token assembly
@gpu
@pytest.mark.parametrize('b,np_,c', VIT)
def test_assemble_tokens_conforms(b, np_, c):
    """saicv_vit_assemble_tokens (fp32 add, bit-exact) and its backward: dpatch = rne(dx), dpos / dcls sum over the batch,
    then a second backward accumulated onto the first (engine/vit.py passes accumulate when the sink holds a gradient)."""
    patch, cls, pos = _randn(b * np_, c, seed=20), _randn(c, seed=21), _randn(np_ + 1, c, seed=22)
    dx1 = _randn(b, np_ + 1, c, seed=23) * (_rand(1, np_ + 1, c, seed=24) * 4)
    dx2 = _randn(b, np_ + 1, c, seed=25)
    what = f'assemble B {b} NP {np_} C {c}'

    def run():
        o = {'x': _nan(b, np_ + 1, c), 'dpos': _nan(np_ + 1, c), 'dcls': _nan(c), 'dpatch': _nanb(b * np_, c),
             'dpatch2': _nanb(b * np_, c)}
        _c('saicv_vit_assemble_tokens', patch, cls, pos, o['x'], b, np_, c)
        _c('saicv_vit_assemble_tokens_bwd', dx1, o['dpos'], o['dcls'], o['dpatch'], b, np_, c, 0)
        o['dpos1'], o['dcls1'] = o['dpos'].clone(), o['dcls'].clone()
        _c('saicv_vit_assemble_tokens_bwd', dx2, o['dpos'], o['dcls'], o['dpatch2'], b, np_, c, 1)
        return o

    o = run()
    src = torch.cat([cls.expand(b, 1, c), patch.view(b, np_, c)], 1)
    _exact('assemble_tokens', f'{what} x', o['x'], (src.double() + pos.double()).float())
    _exact('assemble_tokens_bwd', f'{what} dpatch', o['dpatch'], _bf(dx1[:, 1:].reshape(b * np_, c)))
    _exact('assemble_tokens_bwd', f'{what} dpatch (second call)', o['dpatch2'], _bf(dx2[:, 1:].reshape(b * np_, c)))
    s, a = dx1.double().sum(0), b * U * dx1.double().abs().sum(0)
    _check('assemble_tokens_bwd', f'{what} dpos', o['dpos1'], s, a)
    _same(f'{what} dcls is dpos[0]', o['dcls1'], o['dpos1'][0])
    s2, a2 = dx2.double().sum(0), b * U * dx2.double().abs().sum(0)
    v = o['dpos1'].double() + s2
    _check('assemble_tokens_bwd', f'{what} dpos (accumulate)', o['dpos'], v, _norm._rnd(v, a2))
    v = o['dcls1'].double() + s2[0]
    _check('assemble_tokens_bwd', f'{what} dcls (accumulate)', o['dcls'], v, _norm._rnd(v, a2[0]))
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


# ------------------------------------------------------------------ ViT token pooling
@gpu
@pytest.mark.parametrize('b,l,c,mean,scaled', POOL)
def test_token_pool_conforms(b, l, c, mean, scaled):
    """saicv_token_pool_fwd / _bwd: mean over tokens 1 .. L-1 or the cls token; the backward's fp32 dx and its bf16 copy
    times the next block's drop-path scale (bf16_row_scale, per batch element)."""
    x = _randn(b, l, c, seed=30) * 2 + _randn(1, 1, c, seed=31)
    dp = _randn(b, c, seed=32)
    rs = (_rand(b, seed=33) > 0.25).float() * (_rand(b, seed=34) + 0.5) if scaled else None
    what = f'pool B {b} L {l} C {c} {"mean" if mean else "cls"}{" scaled" if scaled else ""}'

    def run():
        o = {'pooled': _nan(b, c), 'dx': _nan(b, l, c), 'dxb': _nanb(b, l, c)}
        _c('saicv_token_pool_fwd', x, o['pooled'], b, l, c, mean)
        _c('saicv_token_pool_bwd', dp, o['dx'], o['dxb'], rs, b, l, c, mean)
        return o

    o = run()
    zf, zb = torch.zeros(b, c, device='cuda'), torch.zeros(b, c, device='cuda', dtype=BF16)
    r = rs.double()[:, None] if scaled else 1.0
    if mean:
        t = x[:, 1:].double()
        a_s = (l - 1) * U * t.abs().sum(1) / (l - 1)
        v = t.sum(1) / (l - 1)
        del t
        _check('token_pool_fwd', f'{what} pooled', o['pooled'], v, _norm._rnd(v, a_s))
        v = dp.double() / (l - 1)
        a = _norm._rnd(v, U * v.abs())                       # rn(1 / (L - 1)), then the product
        _check('token_pool_bwd', f'{what} dx', o['dx'][:, 1:], v[:, None].expand(b, l - 1, c), a[:, None])
        _exact('token_pool_bwd', f'{what} dx token 0', o['dx'][:, 0], zf)
        w = v * r
        _check('token_pool_bwd', f'{what} dx bf16', o['dxb'][:, 1:], w[:, None].expand(b, l - 1, c),
               _norm._rnd(w, a * r)[:, None])
        _exact('token_pool_bwd', f'{what} dx bf16 token 0', o['dxb'][:, 0], zb)
    else:
        _exact('token_pool_fwd', f'{what} pooled', o['pooled'], x[:, 0])
        _exact('token_pool_bwd', f'{what} dx token 0', o['dx'][:, 0], dp)
        _exact('token_pool_bwd', f'{what} dx tokens 1..', o['dx'][:, 1:], torch.zeros(b, l - 1, c, device='cuda'))
        w = dp.double() * r
        _check('token_pool_bwd', f'{what} dx bf16 token 0', o['dxb'][:, 0], w, U * w.abs())
        _exact('token_pool_bwd', f'{what} dx bf16 tokens 1..', o['dxb'][:, 1:],
               torch.zeros(b, l - 1, c, device='cuda', dtype=BF16))
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


# ------------------------------------------------------------------ MAE token gather / scatter
def _fill_grad(fam, what, dout, idx, dfill):
    """dfill (fp32 [C]) against the exact sum of the dout rows with idx < 0."""
    rows, c = idx.numel(), dout.shape[-1]
    t = dout.reshape(rows, c)[idx.flatten() < 0].double()
    _check(fam, f'{what} dfill', dfill, t.sum(0), _fill_depth(rows) * U * t.abs().sum(0))


def _gather_bwd(dout, idx, src_rows, b, r, c, bf16, dsrc):
    nslab = _fill_slabs(b * r)
    part, dfill = _nan(nslab, c), _nan(c)
    _c('saicv_token_gather_bwd', dout, idx, dsrc, int(bf16), src_rows, part, b, r, c)
    _c('saicv_reduce_partials', part, dfill, nslab, c, 0)
    return dsrc, dfill


def _shuffle(b, n, seed):
    ids_shuffle = _rand(b, n, seed=seed).argsort(1)
    return ids_shuffle, ids_shuffle.argsort(1)


@gpu
@pytest.mark.parametrize('b,c', MAE_ENC)
def test_mae_encoder_gather_conforms(b, c):
    """Encoder: keep 49 of 196 patch tokens, row 0 takes cls_token (idx -1), pos by pos_idx; the backward scatters into
    a pre-zeroed dsrc (unreferenced rows stay 0), fp32 and bf16, and reduces the cls gradient over the fill slabs."""
    n, keep = 196, 49
    r = keep + 1
    ids_keep = _shuffle(b, n, 40)[0][:, :keep]
    minus = torch.full((b, 1), -1, device='cuda', dtype=torch.int64)
    idx = torch.cat([minus, ids_keep], 1).int().contiguous()
    pos_idx = torch.cat([minus + 1, ids_keep + 1], 1).int().contiguous()
    src, cls, pos = _randn(b, n, c, seed=41), _randn(c, seed=42), _randn(n + 1, c, seed=43)
    dout = _randn(b, r, c, seed=44)
    what = f'mae encoder B {b} C {c}'

    def run():
        o = {'out': _nan(b, r, c)}
        _c('saicv_token_gather_fwd', src, n, idx, cls, pos, pos_idx, o['out'], b, r, c)
        for dt in (F32, BF16):
            o[f'dsrc {dt}'], o[f'dfill {dt}'] = _gather_bwd(dout, idx, n, b, r, c, dt == BF16,
                                                            torch.zeros(b, n, c, device='cuda', dtype=dt))
        return o

    o = run()
    rows = torch.cat([cls.expand(b, 1, c), src.gather(1, ids_keep[:, :, None].expand(b, keep, c))], 1)
    _exact('token_gather_fwd', f'{what} out', o['out'], (rows.double() + pos[pos_idx.long()].double()).float())
    ref = torch.zeros(b, n, c, device='cuda').scatter(1, ids_keep[:, :, None].expand(b, keep, c), dout[:, 1:])
    _exact('token_gather_bwd', f'{what} dsrc fp32', o[f'dsrc {F32}'], ref)
    _exact('token_gather_bwd', f'{what} dsrc bf16', o[f'dsrc {BF16}'], _bf(ref))
    for dt in (F32, BF16):
        _fill_grad('token_fill_grad', f'{what} ({dt})', dout, idx, o[f'dfill {dt}'])
        _same(f'{what} dfill does not depend on the dsrc dtype', o[f'dfill {dt}'], o[f'dfill {F32}'])
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


@gpu
@pytest.mark.parametrize('b,c', MAE_DEC)
def test_mae_decoder_unshuffle_conforms(b, c):
    """Decoder: 197 rows from the 50 encoder tokens, idx -1 takes mask_token, pos by row; every source row is referenced
    once, so dsrc is NaN-prefilled (zero=False) and every element must be written.  B = 512 runs the fill gradient at its
    128-slab cap with 788 rows per slab."""
    n, keep = 196, 49
    le, r = keep + 1, n + 1
    restore = _shuffle(b, n, 50)[1]
    idx = torch.cat([torch.zeros(b, 1, device='cuda', dtype=torch.int64),
                     torch.where(restore < keep, restore + 1, -1)], 1).int().contiguous()
    y, mask, pos = _randn(b, le, c, seed=51), _randn(c, seed=52), _randn(r, c, seed=53)
    dout = _randn(b, r, c, seed=54) * (_rand(1, r, 1, seed=55) * 4)
    what = f'mae decoder B {b} C {c}'

    def run():
        o = {'out': _nan(b, r, c)}
        _c('saicv_token_gather_fwd', y, le, idx, mask, pos, None, o['out'], b, r, c)
        for dt in (F32, BF16):
            o[f'dsrc {dt}'], o[f'dfill {dt}'] = _gather_bwd(dout, idx, le, b, r, c, dt == BF16,
                                                            _nan(b, le, c, dtype=dt))
        return o

    o = run()
    il = idx.long()
    rows = torch.where(il[:, :, None] >= 0, y.gather(1, il.clamp_min(0)[:, :, None].expand(b, r, c)), mask)
    _exact('token_gather_fwd', f'{what} out', o['out'], (rows.double() + pos.double()).float())
    # the inverse map: source row s of batch b came from output row src_of[b, s]
    src_of = torch.empty(b, le, device='cuda', dtype=torch.int64)
    live = il >= 0
    src_of[live.nonzero()[:, 0], il[live]] = live.nonzero()[:, 1]
    ref = dout.gather(1, src_of[:, :, None].expand(b, le, c))
    _exact('token_gather_bwd', f'{what} dsrc fp32', o[f'dsrc {F32}'], ref)
    _exact('token_gather_bwd', f'{what} dsrc bf16', o[f'dsrc {BF16}'], _bf(ref))
    for dt in (F32, BF16):
        _fill_grad('token_fill_grad', f'{what} ({dt})', dout, idx, o[f'dfill {dt}'])
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


# ------------------------------------------------------------------ SAM windows and positional embedding
@gpu
@pytest.mark.parametrize('b,h,w,c,ws', WIN)
def test_window_partition_conforms(b, h, w, c, ws):
    """Window partition (padding rows +0) and unpartition (padding rows dropped): 64 x 64 at ws 14 pads to 70 and at
    ws 16 tiles exactly; 20 x 20 pads; 9 x 7 is smaller than one window; 24 x 40 has H != W."""
    nwy, nwx = -(-h // ws), -(-w // ws)
    x = _randb(b, h, w, c, seed=60)
    win = _randb(b * nwy * nwx, ws * ws, c, seed=61)
    what = f'windows B {b} {h}x{w} C {c} ws {ws}'

    def run():
        o = {'win': _nanb(b * nwy * nwx, ws * ws, c), 'x': _nanb(b, h, w, c)}
        _c('saicv_window_partition', x, o['win'], b, h, w, c, ws)
        _c('saicv_window_unpartition', win, o['x'], b, h, w, c, ws)
        return o

    o = run()
    xp = F.pad(x, (0, 0, 0, nwx * ws - w, 0, nwy * ws - h))
    ref = xp.view(b, nwy, ws, nwx, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(b * nwy * nwx, ws * ws, c)
    _exact('window partition', f'{what} partition', o['win'], ref)
    ref = win.view(b, nwy, nwx, ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(b, nwy * ws, nwx * ws, c)[:, :h, :w]
    _exact('window partition', f'{what} unpartition', o['x'], ref.contiguous())
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


@gpu
@pytest.mark.parametrize('b,per', ADDPOS)
def test_add_pos_embed_conforms(b, per):
    """saicv_add_pos_embed: x += pos broadcast over the batch, in place, one fp32 add."""
    x0, pos = _randn(b, per, seed=70) * 2, _randn(per, seed=71) * 0.1

    def run():
        x = x0.clone()
        _c('saicv_add_pos_embed', x, pos, b, per)
        return x

    x = run()
    _exact('add_pos_embed', f'add_pos_embed B {b} per {per}', x, (x0.double() + pos.double()).float())
    _same(f'add_pos_embed B {b} per {per} on a second launch', run(), x)


# ------------------------------------------------------------------ SAM rel-pos score columns
def _grid_index(sh, sw):
    l = torch.arange(sh * sw, device='cuda')
    return l // sw, l % sw


@gpu
@pytest.mark.parametrize('sh,sw,hd,bw,heads', RELPOS)
def test_relpos_kernels_conform(sh, sw, hd, bw, heads):
    """relpos_pack_q, relpos_table, relpos_gather, relpos_shift and relpos_dq_combine at dqk = relpos_dqk and
    nip = relpos_nip.  The (5, 9) grid is the case in which a swap of Sh and Sw in the index maths shows."""
    ops = _ops()
    L = sh * sw
    dqk, nip = ops.relpos_dqk(hd, sh, sw), ops.relpos_nip(sh, sw)
    nh, nw = 2 * sh - 1, 2 * sw - 1
    rows = bw * heads * L
    scale = _f32(hd ** -0.5)
    qkv = _randb(bw, L, 3, heads, hd, seed=80)
    rph, rpw = _randn(nh, hd, seed=81) * 0.1, _randn(nw, hd, seed=82)
    T = _randb(rows, nip, seed=83)
    dqe = _randb(rows, dqk, seed=84)
    dqx = _randn(rows, hd, seed=85)
    what = f'relpos {sh}x{sw} hd {hd} windows {bw} heads {heads}'

    def run():
        o = {'qc': _nanb(rows, hd), 'rtab': _nanb(nip, hd), 'qe': _nanb(rows, dqk), 'ke': _nanb(rows, dqk),
             'ef': _nanb(rows, nip), 'dqkv': _nanb(bw, L, 3, heads, hd)}
        _c('saicv_relpos_pack_q', qkv, o['qc'], bw, heads, hd, L)
        _c('saicv_relpos_table', rph, rpw, o['rtab'], sh, sw, nip, hd)
        _c('saicv_relpos_gather', qkv, T, o['qe'], o['ke'], bw, heads, hd, sh, sw, dqk, nip, scale)
        _c('saicv_relpos_shift', dqe, o['ef'], bw, heads, hd, sh, sw, dqk, nip)
        _c('saicv_relpos_dq_combine', dqe, dqx, o['dqkv'], bw, heads, hd, L, dqk, scale)
        return o

    o = run()
    per_head = lambda t: t.permute(0, 2, 1, 3).reshape(rows, hd)           # noqa: E731  [bw, L, H, hd] -> rows
    q, k = per_head(qkv[:, :, 0]), per_head(qkv[:, :, 1])
    _exact('relpos layout', f'{what} pack_q', o['qc'], q)
    _exact('relpos layout', f'{what} table', o['rtab'],
           _bf(torch.cat([rph, rpw, torch.zeros(nip - nh - nw, hd, device='cuda')])))
    # gather: Qe = [q * scale | T[qh - kh + Sh - 1] | T[nh + qw - kw + Sw - 1] | 0],  Ke = [k | onehot(qh) | onehot(qw) | 0]
    qh, qw = _grid_index(sh, sw)
    col_h = qh[:, None] - torch.arange(sh, device='cuda')[None] + sh - 1
    col_w = nh + qw[:, None] - torch.arange(sw, device='cuda')[None] + sw - 1
    cols = torch.cat([col_h, col_w], 1).expand(bw * heads, L, sh + sw)
    bias = T.view(bw * heads, L, nip).gather(2, cols).reshape(rows, sh + sw)
    pad = torch.zeros(rows, dqk - hd - sh - sw, device='cuda', dtype=BF16)
    v = q.double() * scale
    _check('relpos scale', f'{what} Qe q * scale', o['qe'][:, :hd], v, U * v.abs())
    _exact('relpos layout', f'{what} Qe bias columns', o['qe'][:, hd:], torch.cat([bias, pad], 1))
    onehot = torch.cat([F.one_hot(qh, sh), F.one_hot(qw, sw)], 1).to(BF16).repeat(bw * heads, 1)
    _exact('relpos layout', f'{what} Ke', o['ke'], torch.cat([k, onehot, pad], 1))
    # shift: ef[r][idx] = dT_h[kh] for kh = qh - idx + Sh - 1 in the grid, ef[r][nh + idx] = dT_w[kw], else +0
    idx = torch.arange(nip, device='cuda')[None]
    kh = qh[:, None] - idx + sh - 1
    kw = qw[:, None] - (idx - nh) + sw - 1
    src = torch.where((idx < nh) & (kh >= 0) & (kh < sh), hd + kh,
                      torch.where((idx >= nh) & (idx < nh + nw) & (kw >= 0) & (kw < sw), hd + sh + kw, -1))
    g = dqe.view(bw * heads, L, dqk).gather(2, src.clamp_min(0).expand(bw * heads, L, nip)).reshape(rows, nip)
    ok = (src >= 0).repeat(bw * heads, 1)
    _exact('relpos layout', f'{what} shift', o['ef'], torch.where(ok, g, torch.zeros((), device='cuda', dtype=BF16)))
    # dq_combine: q slot = bf16(fmaf(dqe, scale, dqx)); the k and v slots are not written
    v = dqe[:, :hd].double() * scale + dqx.double()
    _check('relpos scale', f'{what} dq_combine', per_head(o['dqkv'][:, :, 0]), v, U * v.abs())
    _same(f'{what} dq_combine leaves k, v slots', o['dqkv'][:, :, 1:], _nanb(bw, L, 2, heads, hd))
    for key, t in run().items():
        _same(f'{what} {key} on a second launch', t, o[key])


@gpu
def test_relpos_table_wraps():
    """relpos_table with a table far longer than its two tables (only +0 rows past 2 Sh - 1 + 2 Sw - 1), so that its
    grid-stride loop wraps: nip * hd items against one sweep of 540,672."""
    sh, sw, hd, nip = RELPOS_TABLE_WRAP
    rph, rpw = _randn(2 * sh - 1, hd, seed=86), _randn(2 * sw - 1, hd, seed=87)
    rtab = _nanb(nip, hd)
    _c('saicv_relpos_table', rph, rpw, rtab, sh, sw, nip, hd)
    ref = torch.cat([rph, rpw, torch.zeros(nip - rph.shape[0] - rpw.shape[0], hd, device='cuda')])
    _exact('relpos layout', f'relpos table nip {nip} hd {hd}', rtab, _bf(ref))


# ------------------------------------------------------------------ DETR per-head packing
@gpu
@pytest.mark.parametrize('b,l,ldm,colm,tensor_extra,scale', HEADS)
def test_heads_pack_unpack_conform(b, l, ldm, colm, tensor_extra, scale):
    """heads_pack: [B*L, ld] columns col0 + h hd .. -> [B, H, L, dp] scaled, column hd = extra (tensor or constant), rest +0;
    heads_unpack back into the column block of a NaN-filled [B*L, ld] (columns outside it stay NaN)."""
    H, hd, dp = DETR_H, DETR_HD, DETR_DP
    C = H * hd
    ld, col0 = ldm * C, colm * C
    sc = _f32(scale)
    src = _randb(b * l, ld, seed=90, scale=3.0)
    extra = _randn(b * l, seed=91) * 10 if tensor_extra else None
    const = -0.3
    packed = _randb(b, H, l, dp, seed=92)
    what = f'heads B {b} L {l} ld {ld} col0 {col0} {"extra" if tensor_extra else "const"} scale {sc:.6g}'

    def run():
        o = {'dst': _nanb(b, H, l, dp), 'un': _nanb(b * l, ld)}
        _c('saicv_heads_pack', src, ld, col0, extra, const, o['dst'], b, l, H, hd, dp, sc)
        _c('saicv_heads_unpack', packed, o['un'], ld, col0, b, l, H, hd, dp, sc)
        return o

    o = run()
    heads = src.view(b, l, ld)[:, :, col0:col0 + C].view(b, l, H, hd).permute(0, 2, 1, 3)
    if sc == 1.0:
        _exact('heads layout', f'{what} pack', o['dst'][..., :hd], heads)
    else:
        v = heads.double() * sc
        _check('heads scale', f'{what} pack', o['dst'][..., :hd], v, U * v.abs())
    ex = _bf(extra).view(b, 1, l).expand(b, H, l) if tensor_extra else \
        _bf(torch.full((b, H, l), _f32(const), device='cuda', dtype=torch.float64))
    _exact('heads layout', f'{what} pack extra column', o['dst'][..., hd], ex)
    _exact('heads layout', f'{what} pack zero columns', o['dst'][..., hd + 1:],
           torch.zeros(b, H, l, dp - hd - 1, device='cuda', dtype=BF16))
    un = o['un'].view(b, l, ld)
    ref = packed[..., :hd].permute(0, 2, 1, 3).reshape(b, l, C)
    if sc == 1.0:
        _exact('heads layout', f'{what} unpack', un[:, :, col0:col0 + C], ref)
    else:
        v = ref.double() * sc
        _check('heads scale', f'{what} unpack', un[:, :, col0:col0 + C], v, U * v.abs())
    outside = torch.ones(ld, dtype=torch.bool, device='cuda')
    outside[col0:col0 + C] = False
    assert torch.isnan(un[:, :, outside].float()).all(), f'{what}: unpack wrote outside its column block'
    for k, t in run().items():
        _same(f'{what} {k} on a second launch', t, o[k])


# ------------------------------------------------------------------ refusals
def _refusals(f, i):
    """(entry, args without the stream, message fragment); f, i: fp32 / int32 buffers large enough for every shape here,
    so no call could read or write outside them even if it launched."""
    return [
        ('saicv_vit_assemble_tokens', (f, f, f, f, 2, 3, 6), 'C % 4'),
        ('saicv_token_gather_fwd', (f, 4, i, f, f, None, f, 2, 3, 6), 'C % 4'),
        ('saicv_token_gather_bwd', (f, i, f, 0, 4, f, 2, 3, 6), 'C % 4'),
        ('saicv_gelu_fwd', (f, f, 12), 'n % 8'),
        ('saicv_dropout', (f, 1, None, f, 0, f, 1, 16, 0.1, 0, None), 'elems_per_scale'),
        ('saicv_dropout', (f, 1, None, f, 6, f, 1, 16, 0.1, 0, None), 'elems_per_scale'),
        ('saicv_dropout', (f, 1, None, None, 0, f, 1, 18, 0.1, 0, None), 'n % 4'),
        ('saicv_dropout', (f, 1, None, None, 0, f, 1, 16, 1.0, 0, None), 'p must be in'),
        ('saicv_dropout', (f, 1, None, None, 0, f, 1, 16, -0.1, 0, None), 'p must be in'),
        ('saicv_dropout', (f, 1, None, None, 0, f, 1, 16, float('nan'), 0, None), 'p must be in'),
        ('saicv_dropout', (f, 1, f, None, 0, f, 0, 16, 0.1, 0, None), 'residual needs an fp32 output'),
        ('saicv_heads_pack', (f, 64, 0, None, 0.0, f, 1, 2, 2, 32, 32, 1.0), 'dp > hd'),
        ('saicv_heads_pack', (f, 64, 0, None, 0.0, f, 1, 2, 2, 12, 24, 1.0), 'multiples of 8'),
        ('saicv_heads_pack', (f, 64, 4, None, 0.0, f, 1, 2, 2, 16, 24, 1.0), 'multiples of 8'),
        ('saicv_heads_unpack', (f, f, 64, 0, 1, 2, 2, 12, 24, 1.0), 'multiples of 8'),
        ('saicv_window_partition', (f, f, 1, 4, 4, 12, 2), 'C % 8'),
        ('saicv_window_partition', (f, f, 1, 4, 4, 16, 0), 'bad window size'),
        ('saicv_window_unpartition', (f, f, 1, 4, 4, 12, 2), 'C % 8'),
        ('saicv_add_pos_embed', (f, f, 2, 6), 'per-batch size % 4'),
        ('saicv_relpos_pack_q', (f, f, 1, 1, 12, 4), 'hd % 8'),
        ('saicv_relpos_table', (f, f, f, 2, 3, 7, 8), 'nip too small'),
        ('saicv_relpos_gather', (f, f, f, f, 1, 1, 8, 2, 3, 8, 8, 1.0), 'dqk 8 too small'),
        ('saicv_relpos_gather', (f, f, f, f, 1, 1, 8, 2, 3, 16, 4, 1.0), 'nip must be'),
        ('saicv_relpos_gather', (f, f, f, f, 1, 1, 8, 2, 3, 16, 12, 1.0), 'nip must be'),
        ('saicv_relpos_shift', (f, f, 1, 1, 8, 2, 3, 8, 8), 'dqk 8 too small'),
        ('saicv_relpos_shift', (f, f, 1, 1, 8, 2, 3, 16, 0), 'nip must be'),
        ('saicv_relpos_dq_combine', (f, f, f, 1, 1, 12, 4, 16, 1.0), 'hd, dqk must be'),
        ('saicv_relpos_dq_combine', (f, f, f, 1, 1, 8, 4, 12, 1.0), 'hd, dqk must be'),
    ]


@gpu
def test_refusals_launch_nothing():
    """Each C entry's documented refusals (C % 4, n % 8, dp <= hd, nip or dqk too small, a row_scale without
    elems_per_scale, p outside [0, 1), ...) return an error before any kernel is launched."""
    lib = _libmod()
    f = torch.zeros(1 << 20, device='cuda')
    i = torch.zeros(1 << 16, device='cuda', dtype=torch.int32)
    for name, args, msg in _refusals(f, i):
        n0 = lib.launch_count()
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            _c(name, *args)
        assert lib.launch_count() == n0, f'{name}{args[-6:]}: launched before refusing'
    torch.cuda.synchronize()
