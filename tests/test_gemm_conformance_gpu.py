"""Conformance of the GEMM engine (`gemm_sm90_kernel<BN, VAR>`) against a float64 reference, and its bit-identity
invariants.

Reference.  The exact result is computed from the same bf16 operands in float64 on the GPU (matmul, or float64
`F.conv2d` / `conv2d_input` / an im2col matmul for the convolutions), together with the absolute product sum
S = sum_k |a_k b_k| (the same product of |A| and |B|).  The fp32 accumulation may differ from the exact sum by

    B = 2^-16 S + 2^-22 |ref|

(the second term covers a reference that sits next to a bf16 rounding boundary).  The epilogue carries B through its
operations: bias / residual / bf16 addend add one fp32 rounding each, ReLU, the 0/1 masks and the row scale are
1-Lipschitz, dGELU multiplies by gelu'(u) (formula error <= 7e-8 in float64; evaluated in fp32 with the MUFU ex2 / rcp
approximations the factor is off by up to 2.9e-7 on an H100, measured on every bf16 u by
test_dgelu_epilogue_factor_on_every_bf16_input; 4e-7 here).  The result B' is an absolute allowance, never a relative
one: where gelu'(u) is tiny a relative bound would be meaningless.

Measured on an H100 80GB HBM3 (400 W): the accumulation uses at most 6e-7 S, about 5 % of B', in every entry.  Only the
dGELU cases use more, up to 37 % of B', and that share is the gelu' factor's own error above, not the reduction.

Acceptance, for every element (no fraction of misses is allowed):
  * bf16 outputs lie in [rne_bf16(v - B'), rne_bf16(v + B')], v the exact float64 value: the output is a correctly
    rounded bf16 of some value within the fp32 accumulation error of the exact result.  Truncation, a second rounding
    (e.g. the accumulator rounded before the bias add) or a dropped k16 step all fail it;
  * fp32 outputs and split-K partials: |out - v| <= B';
  * fused BatchNorm statistics: the partial rows folded in float64 against float64 sums of the stored bf16 output,
    within 2^-16 sum|y| and 2^-16 sum y^2.
Each check prints max |out - v| / S (for bf16 outputs: the distance from v to the rounding interval of the stored value)
and the largest fraction of B' an element used; run with -s to see them.

Invariants (compared as raw bits).  Every output column is reduced by one m64n64 wgmma per k16 step in k-block order,
whatever the ring depth, the number of staging slices or the tile width, so these must not change any bit:
  * SAICV_GEMM_TUNE over BN in {64, 128} x stages in {2, 3, max} x staging slices in {1, 2, 3}, against the default.
    Fused-statistics partial rows only across settings with the default BN (BN decides which tiles a CTA takes);
  * the aux operand by TMA against SAICV_GEMM_NO_AUX_TMA=1 (per-thread loads);
  * each specialised variant against SAICV_GEMM_FULL_VARIANT=1 (not for the transposed conv weight gradient, which
    refuses it, the phase data gradient and the fused statistics, which ignore it, or the 1-bit mask, which only VAR_AUX
    has);
  * two consecutive launches.
The shapes are ragged (M not a multiple of 128, N not a multiple of 64, reductions not a multiple of 64) and most grids
give CTAs several work items, so slices and stage rings wrap and statistics accumulate over several tiles.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24          # one fp32 rounding, relative
GELU_GRAD_ABS = 4e-7    # |gelu_erf_grad - gelu'| (2.9e-7 measured on every bf16 input)
TUNES = [(bn, st, nb) for bn in (64, 128) for st in (2, 3, 8) for nb in (1, 2, 3)]   # stages 8: as many as fit


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _bf(*shape, scale=1.0, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(*shape, device='cuda', generator=g) * scale).to(torch.bfloat16)


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(*shape, device='cuda', generator=g) * scale


def _pick_bn(n):
    """capi_gemm.cu pick_bn: the tile width with the least padded columns, ties to 128."""
    return 64 if (n + 63) // 64 * 64 < (n + 127) // 128 * 128 else 128


# ------------------------------------------------------------------ the acceptance rule
def _quantum_bf16(x):
    """The bf16 spacing at float64 values x (8 significant bits; subnormal spacing 2^-133), exactly."""
    _, e = torch.frexp(x)
    e = torch.where(x == 0, -200, e.to(torch.int64) - 8)
    return ((e.clamp_min(-133) + 1023) << 52).view(torch.float64)


def _rne_bf16(x):
    """float64 -> nearest bf16 value (ties to even), as float64, in one rounding (x.to(bfloat16) rounds through fp32)."""
    q = _quantum_bf16(x)
    return torch.round(x / q) * q


def _rnd(v, a):
    """Allowance after one fp32 rounding of a value within a of v."""
    return a + U * (v.abs() + a)


def _conform(what, out, v, allow, s):
    """out: kernel output; v: exact float64 value; allow: its allowance B'; s: the absolute product sum."""
    assert out.shape == v.shape, f'{what}: shape {tuple(out.shape)} vs {tuple(v.shape)}'
    o = out.double()
    if out.dtype == torch.bfloat16:
        lo, hi = _rne_bf16(v - allow), _rne_bf16(v + allow)
        bad = (o < lo) | (o > hi)
        dist = ((o - v).abs() - _quantum_bf16(o) / 2).clamp_min(0)   # nearest value that rounds to o (to a factor 2 below a power of 2)
    else:
        bad = (o - v).abs() > allow
        dist = (o - v).abs()
    bad |= ~torch.isfinite(o)
    ratio = (dist / s.clamp_min(1e-30)).max().item()
    used = (dist / allow.clamp_min(1e-300)).max().item()
    print(f'{what}: max |out - ref| / S = {ratio:.3g}, allowance used {used:.3g}')
    n_bad = int(bad.sum())
    if n_bad:
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(
            f'{what}: {n_bad}/{out.numel()} elements outside the allowance; first at flat index {i}: '
            f'out {o.flatten()[i].item():.9g}, exact {v.flatten()[i].item():.9g}, allowance {allow.flatten()[i].item():.3g}')


def _acc_allowance(ref, s):
    return 2.0 ** -16 * s + 2.0 ** -22 * ref.abs()


def _gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x * 0.5 ** 0.5)) + x * torch.exp(-0.5 * x * x) * (2.0 * torch.pi) ** -0.5


def _stats_conform(what, rows, y):
    """Partial rows [r, 2, N] of a fused-statistics GEMM against float64 sums of the stored bf16 output y [M, N]."""
    yd = y.double().view(-1, rows.shape[-1])
    folded = rows.double().sum(0)
    for j, (name, ref, mag) in enumerate((('sum y', yd.sum(0), yd.abs().sum(0)), ('sum y^2', (yd * yd).sum(0), (yd * yd).sum(0)))):
        err = (folded[j] - ref).abs()
        allow = 2.0 ** -16 * mag
        print(f'{what} {name}: max |folded - ref| / sum|.| = {(err / mag.clamp_min(1e-30)).max().item():.3g}, '
              f'allowance used {(err / allow.clamp_min(1e-300)).max().item():.3g}')
        n_bad = int(((err > allow) | ~torch.isfinite(folded[j])).sum())
        assert n_bad == 0, f'{what} {name}: {n_bad}/{err.numel()} columns outside 2^-16 of the absolute sum'


# ------------------------------------------------------------------ the invariants
def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _same(what, a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, f'{what}: {tuple(a.shape)} {a.dtype} vs {tuple(b.shape)} {b.dtype}'
    n_bad = int((_bits(a) != _bits(b)).sum())
    assert n_bad == 0, f'{what}: {n_bad}/{a.numel()} elements differ (max |diff| {(a.float() - b.float()).abs().max().item():.3g})'


def _invariants(monkeypatch, run, base, aux=False, stats_bn=None, full_variant=True):
    """run() -> dict of outputs, base = run() under the defaults.  stats_bn: the default tile width of a
    fused-statistics launch (its 'stats' partial rows are compared only where the tile width is kept)."""
    def compare(setting, got, keep_stats=True):
        for name, ref in base.items():
            if name == 'stats' and not keep_stats:
                continue
            _same(f'{name} under {setting}', got[name], ref)

    compare('a second launch', run())
    for bn, st, nb in TUNES:
        with monkeypatch.context() as m:
            m.setenv('SAICV_GEMM_TUNE', f'{bn}:{st}:{nb}')
            got = run()
        compare(f'SAICV_GEMM_TUNE={bn}:{st}:{nb}', got, keep_stats=stats_bn == bn)
    envs = []
    if aux:
        envs.append('SAICV_GEMM_NO_AUX_TMA')
    if full_variant:
        envs.append('SAICV_GEMM_FULL_VARIANT')
    for env in envs:
        with monkeypatch.context() as m:
            m.setenv(env, '1')
            got = run()
        compare(f'{env}=1', got)


# ------------------------------------------------------------------ float64 references
def _mm64(a, b_t):
    """a [M, K] @ b_t[N, K]^T in float64 and the absolute product sum."""
    a, b_t = a.double(), b_t.double()
    return a @ b_t.t(), a.abs() @ b_t.abs().t()


def test_rne_bf16_reference_rounding():
    """The reference rounding itself (CPU): agrees with torch's fp32 -> bf16 on fp32 values (one rounding there) and
    rounds float64 values that torch would round twice correctly."""
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(100000, generator=g) * 10.0 ** torch.randint(-30, 30, (100000,), generator=g).float(),
                   torch.tensor([0.0, -0.0, 1.0, 1.00390625, 1.01171875, -1.00390625, 2.0 ** -130, 3 * 2.0 ** -134])])
    assert torch.equal(_rne_bf16(x.double()), x.to(torch.bfloat16).double())
    # 1 + 2^-8 is a tie (rounds to even: 1); 1 + 2^-8 + 2^-30 is above it but rounds to the tie in fp32 first
    v = torch.tensor([1 + 2.0 ** -8 + 2.0 ** -30, 1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8 + 2.0 ** -30)], dtype=torch.float64)
    assert _rne_bf16(v).tolist() == [1 + 2.0 ** -7, 1.0, 1 + 2.0 ** -6, -(1 + 2.0 ** -7)]
    assert v.to(torch.bfloat16).double()[0].item() == 1.0   # the double rounding this helper avoids


# ------------------------------------------------------------------ linear forward
LIN_SHAPES = [(300, 72, 8), (1000, 200, 80), (5000, 840, 200), (6000, 328, 1000)]   # M, N, K; the last two: > 132 tiles
LIN_CASES = [(m, *s) for s in LIN_SHAPES for m in ('bf16', 'bias_relu', 'f32_resid_rowscale')]


@pytest.mark.gpu
@pytest.mark.parametrize('mode,M,N,K', LIN_CASES)
def test_linear_fwd_conforms(mode, M, N, K, monkeypatch):
    ops = _ops()
    x, w = _bf(M, K, seed=1), _bf(N, K, scale=K ** -0.5, seed=2)
    bias = _randn(N, scale=0.5, seed=3)
    rps = 197
    resid = _randn(M, N, seed=4)
    scale = torch.rand((M + rps - 1) // rps, device='cuda', generator=torch.Generator(device='cuda').manual_seed(5)) * 2

    def run():
        if mode == 'bf16':
            return {'y': ops.linear_fwd(x, w)}
        if mode == 'bias_relu':
            return {'y': ops.linear_fwd(x, w, bias=bias, flags=ops.EPI_RELU)}
        return {'y': ops.linear_fwd(x, w, bias=bias, resid=resid, out_f32=True, row_scale=scale, rows_per_scale=rps)}

    base = run()
    ref, s = _mm64(x, w)
    a = _acc_allowance(ref, s)
    v = ref
    if mode != 'bf16':
        v = ref + bias.double()
        a = _rnd(v, a)
    if mode == 'bias_relu':
        v = v.clamp_min(0)
    elif mode == 'f32_resid_rowscale':
        sc = scale.double().repeat_interleave(rps)[:M, None]
        v, a = sc * v, sc * a
        a = _rnd(v, a)
        v = v + resid.double()
        a = _rnd(v, a)
    _conform(f'linear_fwd {mode} {M}x{N}x{K}', base['y'], v, a, s)
    del ref, s, a, v
    _invariants(monkeypatch, run, base, aux=mode == 'f32_resid_rowscale')


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K', [(2 * 112 * 112, 64, 192), (20000, 328, 200)])
def test_linear_fwd_fused_statistics_conform(M, N, K, monkeypatch):
    """The explicit-im2col stem GEMM with BatchNorm statistics: 196 tiles at the stem's shape, 471 at the ragged one.  The
    column-tile counts (1 and 3, or 6 at BN = 64) divide 132, so the CTAs of a full H100 meet the same columns again and
    add several tiles into one accumulator (with 7 column tiles, say, a CTA would see each column at most once per
    924 work items), and they cycle the stats warps' slice ring."""
    ops = _ops()
    x, w = _bf(M, K, seed=6), _bf(N, K, scale=K ** -0.5, seed=7)

    def run():
        rows = ops.gemm_stats_rows(M, N)
        ws = torch.full((rows, 2, N), float('nan'), device='cuda')
        y = ops.linear_fwd(x, w, stats=ws)
        return {'y': y, 'stats': ws}

    base = run()
    ref, s = _mm64(x, w)
    _conform(f'linear_fwd stats {M}x{N}x{K}', base['y'], ref, _acc_allowance(ref, s), s)
    del ref, s
    _stats_conform(f'linear_fwd stats {M}x{N}x{K}', base['stats'], base['y'])
    _invariants(monkeypatch, run, base, stats_bn=_pick_bn(N), full_variant=False)


# ------------------------------------------------------------------ linear data gradient
DG_SHAPES = [(300, 8, 72), (1000, 80, 200), (5000, 200, 840), (6000, 1000, 328)]   # M, N (reduction), K (output columns)
DG_MODES = ['bf16', 'f32_resid', 'add', 'relu_out', 'gelu_pre', 'f32_resid_gelu_pre']


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K', DG_SHAPES)
@pytest.mark.parametrize('mode', DG_MODES)
def test_linear_dgrad_conforms(mode, M, N, K, monkeypatch):
    """dx[M, K] = dy[M, N] w[N, K] with each epilogue operand.  The fp32 residual plus a bf16 operand ('both': per-thread
    loads, VAR_FULL) computes (dy w + resid) * gelu'(u)."""
    ops = _ops()
    dy, w = _bf(M, N, seed=8), _bf(N, K, scale=N ** -0.5, seed=9)
    aux = _bf(M, K, scale=2.0, seed=10)
    resid = _randn(M, K, seed=11)

    def run():
        if mode == 'bf16':
            return {'dx': ops.linear_dgrad(dy, w)}
        if mode == 'f32_resid':
            return {'dx': ops.linear_dgrad(dy, w, resid=resid, out_f32=True)}
        if mode == 'add':
            return {'dx': ops.linear_dgrad(dy, w, add=aux)}
        if mode == 'relu_out':
            return {'dx': ops.linear_dgrad(dy, w, relu_out=aux)}
        if mode == 'gelu_pre':
            return {'dx': ops.linear_dgrad(dy, w, gelu_pre=aux)}
        return {'dx': ops.linear_dgrad(dy, w, resid=resid, out_f32=True, gelu_pre=aux)}

    base = run()
    ref, s = _mm64(dy, w.t())
    a = _acc_allowance(ref, s)
    v = ref
    u = aux.double()
    if mode in ('f32_resid', 'f32_resid_gelu_pre'):
        v = v + resid.double()
        a = _rnd(v, a)
    if mode == 'add':
        v = v + u
        a = _rnd(v, a)
    elif mode == 'relu_out':
        keep = (u > 0).double()
        v, a = v * keep, a * keep
    elif mode in ('gelu_pre', 'f32_resid_gelu_pre'):
        g = _gelu_grad64(u)
        a = g.abs() * a + GELU_GRAD_ABS * (v.abs() + a)
        v = v * g
        a = _rnd(v, a)
    _conform(f'linear_dgrad {mode} {M}x{N}x{K}', base['dx'], v, a, s)
    del ref, s, a, v
    _invariants(monkeypatch, run, base, aux=mode != 'bf16')


@pytest.mark.gpu
def test_dgelu_epilogue_factor_on_every_bf16_input():
    """gelu_erf_grad as the epilogue applies it, on every finite bf16 pre-activation: with dy = 0 and an fp32 residual of
    1, the fp32 output of the 'both' data gradient is (0 + 1) * gelu_erf_grad(u) exactly.  Its distance from the exact
    gelu'(u) is the GELU_GRAD_ABS term of the dGELU allowance, which dominates what those cases use of it."""
    ops = _ops()
    u = torch.arange(-2 ** 15, 2 ** 15, device='cuda', dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    u = u[torch.isfinite(u.float())]
    u = torch.cat([u, u.new_zeros((-u.numel()) % 256)]).view(-1, 256).contiguous()
    M, K = u.shape
    dy, w = torch.zeros(M, 64, device='cuda', dtype=torch.bfloat16), _bf(64, K, seed=26)
    g = ops.linear_dgrad(dy, w, resid=torch.ones(M, K, device='cuda'), out_f32=True, gelu_pre=u)
    err = (g.double() - _gelu_grad64(u.double())).abs()
    worst = int(err.argmax())
    print(f'gelu_erf_grad: max |error| {err.max().item():.3g} at u = {u.flatten()[worst].item():.6g} '
          f'(allowance term {GELU_GRAD_ABS:.3g})')
    assert err.max().item() <= GELU_GRAD_ABS


# ------------------------------------------------------------------ weight gradients (split-K partials)
def _split_rows(total, splits):
    """Reduction rows [lo, hi) of each split: saicv_*_wgrad give each split ceil(blocks / splits) 64-row blocks."""
    blocks = (total + 63) // 64
    per = (blocks + splits - 1) // splits
    return [(j * per * 64, min((j + 1) * per * 64, total)) for j in range(splits)]


def _linear_wgrad(dy, x, splits, transposed):
    """ops.linear_wgrad with the split count fixed (ops picks it from the tile width, which SAICV_GEMM_TUNE changes)."""
    from simpleaicv_pytorch_training_examples_b200 import _lib
    ops = _ops()
    M, N = dy.shape
    K = x.shape[1]
    a, b, rows, cols = (x, dy, K, N) if transposed else (dy, x, N, K)
    part = torch.empty(splits, rows, cols, device='cuda')
    _lib.call('saicv_linear_wgrad', ops._p(a), ops._p(b), ops._p(part), M, rows, cols, splits, ops._stream())
    return part


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K,transposed', [(2100, 256, 200, False), (2100, 64, 200, True), (19700, 768, 768, False),
                                              (19700, 768, 768, True)])
def test_linear_wgrad_partials_conform(M, N, K, transposed, monkeypatch):
    """Each split's partial dW = dy[rows]^T x[rows] on its own (M = 2 x 25 x 42 DETR tokens and 100 x 197 ViT tokens:
    the last 64-row block of the last split is ragged)."""
    ops = _ops()
    dy, x = _bf(M, N, scale=M ** -0.5, seed=12), _bf(M, K, seed=13)
    splits = ops.wgrad_splits(N, K, M)
    assert splits > 1

    def run():
        p = _linear_wgrad(dy, x, splits, transposed)
        return {'partials': p.transpose(1, 2).contiguous() if transposed else p}

    base = run()
    for j, (lo, hi) in enumerate(_split_rows(M, splits)):
        ref, s = _mm64(dy[lo:hi].t(), x[lo:hi].t())
        _conform(f'linear_wgrad{"^T" if transposed else ""} {M}x{N}x{K} split {j}/{splits}', base['partials'][j], ref,
                 _acc_allowance(ref, s), s)
    _invariants(monkeypatch, run, base)


def _conv_operands(n, h, w, c, k, r, stride, pad, seed, x_scale=1.0):
    """x NHWC bf16, weights [k, c, r, r] bf16 and their GEMM layout [k, r*r*c] (taps outer, channels inner)."""
    x = _bf(n, h, w, c, scale=x_scale, seed=seed)
    wt = _bf(k, c, r, r, scale=(c * r * r) ** -0.5, seed=seed + 1)
    wb = wt.permute(0, 2, 3, 1).reshape(k, r * r * c).contiguous()
    return x, wt, wb, _ops().make_conv_shape(n, h, w, c, k, r, r, stride, pad)


def _patches64(x, r, stride, pad):
    """im2col of NHWC x in float64: [n*P*Q, r*r*c], column (tap, channel) as in the weight matrix."""
    n, h, w, c = x.shape
    cols = F.unfold(x.double().permute(0, 3, 1, 2), r, padding=pad, stride=stride)       # [n, c*r*r, P*Q]
    return cols.view(n, c, r * r, -1).permute(0, 3, 2, 1).reshape(-1, r * r * c)


def _conv_wgrad(dy, x, cs, splits):
    """ops.conv_wgrad with the split count fixed; partials as [splits, k, r*r*c] whichever orientation ran."""
    from simpleaicv_pytorch_training_examples_b200 import _lib
    ops = _ops()
    ncols = cs.r * cs.s * cs.c
    tr = ops.wgrad_transposed(cs.k, ncols)
    part = torch.empty((splits, ncols, cs.k) if tr else (splits, cs.k, ncols), device='cuda')
    _lib.call('saicv_conv_wgrad', ops._p(dy), ops._p(x), ops._p(part), ctypes.byref(cs), splits, ops._stream())
    return part.transpose(1, 2).contiguous() if tr else part


@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', [
    (5, 30, 30, 128, 256, 3, 1, 1),    # dW, 4500 pixels: ragged last block
    (5, 30, 30, 64, 64, 3, 1, 1),      # dW^T (few filters: A is the im2col patch tile, MN-major)
    (4, 30, 30, 256, 64, 1, 1, 0),     # dW^T, 1x1
    (8, 29, 29, 128, 256, 3, 2, 1),    # dW, stride 2, 1800 pixels
])
def test_conv_wgrad_partials_conform(n, h, w, c, k, r, stride, pad, monkeypatch):
    ops = _ops()
    x, _, _, cs = _conv_operands(n, h, w, c, k, r, stride, pad, seed=14)
    P, Q = ops.conv_out_size(h, pad, r, stride), ops.conv_out_size(w, pad, r, stride)
    pix = n * P * Q
    dy = _bf(n, P, Q, k, scale=pix ** -0.5, seed=16)
    ncols = r * r * c
    splits = ops.wgrad_splits(k, ncols, pix)
    assert splits > 1 and pix % 64
    tr = ops.wgrad_transposed(k, ncols)

    def run():
        return {'partials': _conv_wgrad(dy, x, cs, splits)}

    base = run()
    cols = _patches64(x, r, stride, pad)
    dyd = dy.double().view(pix, k)
    for j, (lo, hi) in enumerate(_split_rows(pix, splits)):
        ref, s = dyd[lo:hi].t() @ cols[lo:hi], dyd[lo:hi].abs().t() @ cols[lo:hi].abs()
        _conform(f'conv_wgrad{"^T" if tr else ""} {n}x{h}x{w} c{c} k{k} r{r} s{stride} split {j}/{splits}',
                 base['partials'][j], ref, _acc_allowance(ref, s), s)
    del cols
    _invariants(monkeypatch, run, base, full_variant=not tr)


# ------------------------------------------------------------------ convolution forward with statistics
@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', [
    (32, 56, 56, 64, 64, 3, 1, 1),     # ResNet layer1 at batch 32: 784 tiles, ~6 per CTA
    (32, 56, 56, 64, 256, 1, 1, 0),    # 1568 tiles
    (7, 29, 29, 128, 192, 3, 1, 1),    # ragged M and N (BN = 64 by default, 128 under SAICV_GEMM_TUNE)
])
def test_conv_fprop_fused_statistics_conform(n, h, w, c, k, r, stride, pad, monkeypatch):
    """Output and BatchNorm partial rows of conv_fprop(stats=), taken by the stats warps."""
    ops = _ops()
    x, wt, wb, cs = _conv_operands(n, h, w, c, k, r, stride, pad, seed=17)
    M = n * ops.conv_out_size(h, pad, r, stride) * ops.conv_out_size(w, pad, r, stride)

    def run():
        ws = torch.full((ops.gemm_stats_rows(M, k), 2, k), float('nan'), device='cuda')
        y = ops.conv_fprop(x, wb, cs, stats=ws)
        return {'y': y, 'stats': ws}

    base = run()
    xd = x.double().permute(0, 3, 1, 2)
    ref = F.conv2d(xd, wt.double(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    s = F.conv2d(xd.abs(), wt.double().abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    what = f'conv_fprop stats {n}x{h}x{w} c{c} k{k} r{r}'
    _conform(what, base['y'], ref, _acc_allowance(ref, s), s)
    del xd, ref, s
    _stats_conform(what, base['stats'], base['y'])
    _invariants(monkeypatch, run, base, stats_bn=_pick_bn(k), full_variant=False)


# ------------------------------------------------------------------ convolution data gradient
@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w,c,k,r,pad', [(7, 29, 29, 192, 128, 3, 1), (4, 57, 57, 256, 64, 1, 0)])
@pytest.mark.parametrize('mask', [False, True])
def test_conv_dgrad_add_conforms(n, h, w, c, k, r, pad, mask, monkeypatch):
    """Stride 1 with the shortcut gradient added in the epilogue, and multiplied by a 1-bit ReLU mask (ragged M, more
    than 132 tiles)."""
    ops = _ops()
    _, wt, wb, cs = _conv_operands(n, h, w, c, k, r, 1, pad, seed=18)
    dy = _bf(n, h, w, k, seed=20)
    add = _bf(n, h, w, c, seed=21)
    bits = torch.randint(-2 ** 31, 2 ** 31, (n * h * w, c // 32), device='cuda', dtype=torch.int32,
                         generator=torch.Generator(device='cuda').manual_seed(22)) if mask else None

    def run():
        return {'dx': ops.conv_dgrad(dy, wb, cs, add=add, mask_bits=bits)}

    base = run()
    dyd = dy.double().permute(0, 3, 1, 2)
    shape = (n, c, h, w)
    ref = torch.nn.grad.conv2d_input(shape, wt.double(), dyd, padding=pad).permute(0, 2, 3, 1)
    s = torch.nn.grad.conv2d_input(shape, wt.double().abs(), dyd.abs(), padding=pad).permute(0, 2, 3, 1)
    v = ref + add.double()
    a = _rnd(v, _acc_allowance(ref, s))
    if mask:
        b = bits.view(torch.uint8).long()          # little-endian: byte j of a word holds channels 8j .. 8j+7 of it
        keep = ((b.unsqueeze(-1) >> torch.arange(8, device='cuda')) & 1).reshape(n, h, w, c).double()
        v, a = v * keep, a * keep
    _conform(f'conv_dgrad add{"+mask" if mask else ""} {n}x{h}x{w} c{c} k{k} r{r}', base['dx'], v, a, s)
    del dyd, ref, s, v, a
    # the 1-bit mask needs the TMA aux operand in VAR_AUX: neither override applies to it
    _invariants(monkeypatch, run, base, aux=not mask, full_variant=not mask)


@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w,c,k', [(10, 30, 30, 192, 64), (18, 30, 30, 128, 128)])
def test_conv_dgrad_phases_conform(n, h, w, c, k, monkeypatch):
    """3x3 stride-2 data gradient by output phase (Q = 15: tiles of 8 dy rows, 120 of 128 rows; > 132 work items)."""
    ops = _ops()
    _, wt, wb, cs = _conv_operands(n, h, w, c, k, 3, 2, 1, seed=23)
    assert ops.phase_dgrad_ok(cs)
    dy = _bf(n, h // 2, w // 2, k, seed=25)

    def run():
        return {'dx': ops.conv_dgrad(dy, wb, cs)}

    base = run()
    dyd = dy.double().permute(0, 3, 1, 2)
    shape = (n, c, h, w)
    ref = torch.nn.grad.conv2d_input(shape, wt.double(), dyd, stride=2, padding=1).permute(0, 2, 3, 1)
    s = torch.nn.grad.conv2d_input(shape, wt.double().abs(), dyd.abs(), stride=2, padding=1).permute(0, 2, 3, 1)
    _conform(f'conv_dgrad phases {n}x{h}x{w} c{c} k{k}', base['dx'], ref, _acc_allowance(ref, s), s)
    del dyd, ref, s
    _invariants(monkeypatch, run, base, full_variant=False)
