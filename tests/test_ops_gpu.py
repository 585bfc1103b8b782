"""GPU parity of every kernel behind the C ABI against plain torch fp32 on the same inputs.

Inputs are bf16-representable so the only differences are accumulation order (fp32) and the
final bf16 rounding of outputs; tolerances are stated per test.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _bf(*shape, scale=1.0, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(*shape, device='cuda', generator=g) * scale).to(torch.bfloat16)


def _close(got, ref, rtol, atol, what, max_bad_frac=0.0):
    got = got.float()
    ref = ref.float()
    assert got.shape == ref.shape, f'{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad <= max_bad_frac * err.numel(), (
        f'{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, '
        f'ref max {ref.abs().max().item():.4g}')


# ------------------------------------------------------------------ dense layers
@pytest.mark.parametrize('direct', [True, False])
@pytest.mark.parametrize('M,N,K', [(256, 128, 64), (300, 1000, 2048), (1024, 768, 768), (4096, 64, 192)])
def test_linear_fwd(M, N, K, direct):
    ops = _ops()
    x, w = _bf(M, K, seed=1), _bf(N, K, scale=K ** -0.5, seed=2)
    bias = torch.randn(N, device='cuda')
    y = ops.linear_fwd(x, w, bias=bias, flags=ops.EPI_DIRECT if direct else 0)
    ref = x.float() @ w.float().t() + bias
    _close(y, ref, 1e-2, 1e-2, f'linear_fwd bf16 direct={direct}')
    y32 = ops.linear_fwd(x, w, bias=bias, flags=ops.EPI_DIRECT if direct else 0, out_f32=True)
    _close(y32, ref, 1e-4, 1e-4, f'linear_fwd f32 direct={direct}')


def test_linear_fwd_gelu_resid():
    ops = _ops()
    M, N, K = 512, 256, 128
    x, w = _bf(M, K, seed=1), _bf(N, K, scale=K ** -0.5, seed=2)
    bias = torch.randn(N, device='cuda')
    resid = torch.randn(M, N, device='cuda')
    y = ops.linear_fwd(x, w, bias=bias, flags=ops.EPI_GELU)
    _close(y, F.gelu(x.float() @ w.float().t() + bias), 1e-2, 1e-2, 'gelu epilogue')
    y = ops.linear_fwd(x, w, bias=bias, resid=resid, out_f32=True)
    _close(y, x.float() @ w.float().t() + bias + resid, 1e-4, 1e-4, 'residual epilogue')


def test_linear_epilogue_rowscale_and_dgelu():
    ops = _ops()
    M, N, K, L = 6 * 50, 256, 128, 50
    x, w = _bf(M, K, seed=1), _bf(N, K, scale=K ** -0.5, seed=2)
    bias, resid = torch.randn(N, device='cuda'), torch.randn(M, N, device='cuda')
    rs = torch.tensor([0., 1.25, 1.25, 0., 1.25, 1.25], device='cuda')
    y = ops.linear_fwd(x, w, bias=bias, resid=resid, out_f32=True, row_scale=rs, rows_per_scale=L)
    ref = resid + rs.repeat_interleave(L)[:, None] * (x.float() @ w.float().t() + bias)
    _close(y, ref, 1e-4, 1e-4, 'row-scaled residual epilogue')
    dy, u = _bf(M, N, seed=3), _bf(M, K, scale=2.0, seed=4)
    dx = ops.linear_dgrad(dy, w, gelu_pre=u)
    uf = u.float().requires_grad_(True)
    F.gelu(uf).backward(dy.float() @ w.float())
    _close(dx, uf.grad, 1e-2, 1e-2, 'dgelu epilogue')


@pytest.mark.parametrize('tune', ['', '0:0:1', '0:0:2', '0:0:3', '128:3:3', '64:2:2', '192:0:2', 'legacy'])
@pytest.mark.parametrize('M,N,K', [(300, 200, 64), (5000, 768, 256), (1111, 1000, 1024)])
def test_epilogue_aux_operand_by_tma(M, N, K, tune, monkeypatch):
    """The aux operand of the epilogue (fp32 residual / bf16 addend, ReLU mask, GELU pre-activation) is TMA-loaded into the
    staging slices (gemm_sm90.cuh, aux_tma) with 1-3 slices per half and any tile width: ragged M and N, several tiles per
    CTA so the slices wrap, compared with torch and with the per-thread-load path ('legacy')."""
    ops = _ops()
    if tune == 'legacy':
        monkeypatch.setenv('SAICV_GEMM_NO_AUX_TMA', '1')
    elif tune:
        monkeypatch.setenv('SAICV_GEMM_TUNE', tune)
    x, w = _bf(M, K, seed=1), _bf(N, K, scale=K ** -0.5, seed=2)
    bias, resid = torch.randn(N, device='cuda'), torch.randn(M, N, device='cuda')
    lin = x.float() @ w.float().t() + bias
    y = ops.linear_fwd(x, w, bias=bias, resid=resid, out_f32=True)
    _close(y, lin + resid, 1e-4, 1e-4, f'fp32 residual by TMA [{tune}]')
    inplace = resid.clone()
    ops.linear_fwd(x, w, bias=bias, resid=inplace, out_f32=True, out=inplace)
    _close(inplace, lin + resid, 1e-4, 1e-4, f'fp32 residual in place [{tune}]')
    dy, wd = _bf(M, K, seed=3), _bf(K, N, scale=K ** -0.5, seed=4)      # dx[M, N] = dy[M, K] wd[K, N]
    aux = _bf(M, N, scale=2.0, seed=5)
    base = dy.float() @ wd.float()
    _close(ops.linear_dgrad(dy, wd, add=aux), base + aux.float(), 1e-2, 1e-2, f'bf16 addend [{tune}]')
    _close(ops.linear_dgrad(dy, wd, relu_out=aux), base * (aux.float() > 0), 1e-2, 1e-2, f'ReLU mask [{tune}]')
    uf = aux.float().requires_grad_(True)
    F.gelu(uf).backward(base)
    _close(ops.linear_dgrad(dy, wd, gelu_pre=aux), uf.grad, 1e-2, 1e-2, f'dGELU [{tune}]')
    r32 = torch.randn(M, N, device='cuda')
    _close(ops.linear_dgrad(dy, wd, resid=r32, out_f32=True), base + r32, 1e-4, 1e-4, f'fp32 chained gradient [{tune}]')
    # plain outputs through 1-3 staging slices (no aux): bf16 and fp32
    _close(ops.linear_fwd(x, w, bias=bias), lin, 1e-2, 1e-2, f'plain bf16 [{tune}]')
    _close(ops.linear_fwd(x, w, bias=bias, out_f32=True), lin, 1e-4, 1e-4, f'plain fp32 [{tune}]')


@pytest.mark.parametrize('M,N,K', [(256, 128, 64), (300, 1000, 2048), (1024, 3072, 768)])
def test_linear_dgrad(M, N, K):
    ops = _ops()
    dy, w = _bf(M, N, seed=3), _bf(N, K, scale=N ** -0.5, seed=4)
    dx = ops.linear_dgrad(dy, w)
    _close(dx, dy.float() @ w.float(), 1e-2, 1e-2, 'linear_dgrad')


@pytest.mark.parametrize('M,N,K', [(256, 128, 64), (300, 1000, 2048), (50432, 768, 768), (8192, 64, 192)])
def test_linear_wgrad(M, N, K):
    ops = _ops()
    dy, x = _bf(M, N, scale=M ** -0.5, seed=5), _bf(M, K, seed=6)
    part = ops.linear_wgrad(dy, x)
    dw = torch.empty(N, K, device='cuda')
    ops.reduce_partials(part, dw)
    _close(dw, dy.float().t() @ x.float(), 1e-3, 1e-3, f'linear_wgrad splits={part.shape[0]}')


# ------------------------------------------------------------------ convolutions
def _conv_case(n, h, w, c, k, r, stride, pad):
    ops = _ops()
    x_nchw = _bf(n, c, h, w, seed=7).float()
    wt = _bf(k, c, r, r, scale=(c * r * r) ** -0.5, seed=8).float()
    x = x_nchw.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    kpad = r * r * c
    wb = torch.empty(k, kpad, device='cuda', dtype=torch.bfloat16)
    ops.prep_conv_weight(wt.contiguous(), wb, kpad)
    cs = ops.make_conv_shape(n, h, w, c, k, r, r, stride, pad)
    return ops, x_nchw, wt, x, wb, cs


CONV_CASES = [
    (2, 8, 8, 64, 64, 1, 1, 0),
    (2, 8, 8, 64, 64, 3, 1, 1),
    (4, 14, 14, 128, 256, 3, 1, 1),
    (3, 56, 56, 64, 64, 3, 1, 1),
    (4, 28, 28, 128, 128, 3, 2, 1),
    (4, 28, 28, 256, 512, 1, 2, 0),
    (5, 7, 7, 512, 512, 3, 1, 1),
    (2, 16, 16, 64, 128, 3, 2, 1),
]


@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', CONV_CASES)
def test_conv_fprop(n, h, w, c, k, r, stride, pad):
    ops, x_nchw, wt, x, wb, cs = _conv_case(n, h, w, c, k, r, stride, pad)
    y = ops.conv_fprop(x, wb, cs)
    ref = F.conv2d(x_nchw, wt, stride=stride, padding=pad).permute(0, 2, 3, 1)
    _close(y, ref, 1e-2, 1e-2, 'conv_fprop')


@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', CONV_CASES + [(6, 14, 14, 256, 1024, 1, 1, 0), (3, 7, 7, 512, 2048, 1, 1, 0),
                                                       (32, 56, 56, 64, 64, 3, 1, 1), (32, 56, 56, 64, 256, 1, 1, 0)])
def test_conv_fprop_fused_bn_statistics(n, h, w, c, k, r, stride, pad):
    """The GEMM epilogue's per-CTA column sums, folded by bn_finalize, equal the statistics of the
    stored bf16 output (mean rtol 1e-3 / atol 1e-4, rstd rtol 1e-3).  The last two shapes have 784 and 1568 tiles, so
    every CTA adds several tiles into its accumulators."""
    ops, x_nchw, wt, x, wb, cs = _conv_case(n, h, w, c, k, r, stride, pad)
    ws = ops.partial_ws(x.device, 2 * k)
    y = ops.conv_fprop(x, wb, cs, stats=ws)
    rows = y.numel() // k
    gamma, beta = torch.ones(k, device='cuda'), torch.zeros(k, device='cuda')
    ss, saved = torch.empty(2, k, device='cuda'), torch.empty(2, k, device='cuda')
    ops.bn_finalize(ws, gamma, beta, None, None, ss, saved, rows, 1e-5, 0.1, partial_rows=ops.gemm_stats_rows(rows, k))
    yf = y.float().view(rows, k)
    _close(saved[0], yf.mean(0), 1e-3, 1e-4, 'fused mean')
    _close(saved[1], torch.rsqrt(yf.var(0, unbiased=False) + 1e-5), 1e-3, 1e-4, 'fused rstd')
    ref = F.conv2d(x_nchw, wt, stride=stride, padding=pad).permute(0, 2, 3, 1)
    _close(y, ref, 1e-2, 1e-2, 'conv_fprop with stats')


@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', CONV_CASES)
def test_conv_dgrad(n, h, w, c, k, r, stride, pad):
    ops, x_nchw, wt, x, wb, cs = _conv_case(n, h, w, c, k, r, stride, pad)
    P, Q = ops.conv_out_size(h, pad, r, stride), ops.conv_out_size(w, pad, r, stride)
    dy_nchw = _bf(n, k, P, Q, seed=9).float()
    dy = dy_nchw.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    ref = torch.nn.grad.conv2d_input(x_nchw.shape, wt, dy_nchw, stride=stride, padding=pad).permute(0, 2, 3, 1)
    if stride == 1:
        add = _bf(n, h, w, c, seed=23)
        dx = ops.conv_dgrad(dy, wb, cs, add=add)
        ref = ref + add.float()
    elif r == 1:
        # 1x1 stride 2: compact GEMM + strided scatter-add
        dd = ops.linear_dgrad(dy.view(-1, k), wb).view(n, P, Q, c)
        dx = torch.zeros(n, h, w, c, device='cuda', dtype=torch.bfloat16)
        ops.add_strided2(dx, dd)
    else:
        u = ops.zero_upsample2(dy, h, w)
        cs1 = ops.make_conv_shape(n, h, w, c, k, r, r, 1, pad)
        dx = ops.conv_dgrad(u, wb, cs1)
    _close(dx, ref, 1e-2, 2e-2, 'conv_dgrad')


@pytest.mark.parametrize('n,h,w,c,k,r,stride,pad', CONV_CASES)
def test_conv_wgrad(n, h, w, c, k, r, stride, pad):
    ops, x_nchw, wt, x, wb, cs = _conv_case(n, h, w, c, k, r, stride, pad)
    P, Q = ops.conv_out_size(h, pad, r, stride), ops.conv_out_size(w, pad, r, stride)
    dy_nchw = (_bf(n, k, P, Q, seed=10).float() * (n * P * Q) ** -0.5).to(torch.bfloat16).float()
    dy = dy_nchw.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    part = ops.conv_wgrad(dy, x, cs)
    dw = torch.empty(k, c, r, r, device='cuda')
    ops.finish_conv_wgrad(part, dw, r * r * c)
    ref = torch.nn.grad.conv2d_weight(x_nchw, wt.shape, dy_nchw, stride=stride, padding=pad)
    _close(dw, ref, 1e-3, 1e-3, f'conv_wgrad splits={part.shape[0]}')


@pytest.mark.parametrize('n,c,h,w,k,r,stride,pad,kpad', [(4, 3, 32, 32, 64, 7, 2, 3, 192), (3, 3, 37, 41, 64, 3, 1, 1, 128),
                                                       (2, 3, 64, 64, 128, 16, 16, 0, 768), (2, 3, 224, 224, 64, 7, 2, 3, 192),
                                                       (2, 3, 56, 56, 32, 7, 4, 3, 192)])
def test_stem_im2col_matches_conv(n, c, h, w, k, r, stride, pad, kpad):
    ops = _ops()
    assert kpad == ops.stem_kpad(c, r, r)                # filter rows padded to 8 columns, total rounded up to 64
    x = _bf(n, c, h, w, seed=11).float()
    wt = _bf(k, c, r, r, scale=0.1, seed=12).float()
    cols = ops.stem_im2col(x, r, r, stride, pad, kpad)
    wb = torch.empty(k, kpad, device='cuda', dtype=torch.bfloat16)
    ops.prep_conv_weight(wt.contiguous(), wb, kpad, order=ops.ORDER_CRS)
    y = ops.linear_fwd(cols, wb)
    P = ops.conv_out_size(h, pad, r, stride)
    ref = F.conv2d(x, wt, stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(-1, k)
    _close(y, ref, 1e-2, 1e-2, 'stem conv via im2col')
    # weight gradient through the same matrix
    P2 = ops.conv_out_size(w, pad, r, stride)
    dy = _bf(n * P * P2, k, scale=0.05, seed=13)
    part = ops.linear_wgrad(dy, cols)
    dwp = torch.empty(1, k, kpad, device='cuda')
    ops.reduce_partials(part, dwp[0])
    dw = torch.empty(k, c, r, r, device='cuda')
    ops.finish_conv_wgrad(dwp, dw, kpad, order=ops.ORDER_CRS)
    ref_dw = torch.nn.grad.conv2d_weight(x, wt.shape, dy.float().view(n, P, P2, k).permute(0, 3, 1, 2), stride=stride, padding=pad)
    _close(dw, ref_dw, 1e-3, 1e-3, 'stem wgrad')


# ------------------------------------------------------------------ batch norm / pooling
@pytest.mark.parametrize('rows,c', [(4096, 64), (1000, 256), (333, 2048), (50000, 128)])
def test_bn_forward_backward(rows, c):
    ops = _ops()
    y = (_bf(rows, c, seed=14).float() * 2 + 0.5).to(torch.bfloat16)
    res = _bf(rows, c, seed=15)
    gamma = torch.rand(c, device='cuda') + 0.5
    beta = torch.randn(c, device='cuda')
    rmean, rvar = torch.zeros(c, device='cuda'), torch.ones(c, device='cuda')
    stats = torch.zeros(2, c, device='cuda')
    ss, saved = torch.empty(2, c, device='cuda'), torch.empty(2, c, device='cuda')
    part = ops.bn_stats(y)
    ops.bn_finalize(part, gamma, beta, rmean, rvar, ss, saved, rows, 1e-5, 0.1)
    out = torch.empty_like(y)
    ops.bn_apply(y, ss, out, 1, res=res)
    # torch reference (fp32 on the same bf16 inputs)
    yf = y.float().requires_grad_(True)
    resf = res.float().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    rm, rv = torch.zeros(c, device='cuda'), torch.ones(c, device='cuda')
    ref = F.relu(F.batch_norm(yf, rm, rv, g, b, True, 0.1, 1e-5) + resf)
    _close(out, ref, 1e-2, 1e-2, 'bn_apply')
    _close(rmean, rm, 1e-4, 1e-5, 'running_mean')
    _close(rvar, rv, 1e-3, 1e-5, 'running_var')
    dout = _bf(rows, c, seed=16)
    ref.backward(dout.float())
    sums = torch.zeros(2, c, device='cuda')
    dy, dres = torch.empty_like(y), torch.empty_like(y)
    dgamma, dbeta = torch.empty(c, device='cuda'), torch.empty(c, device='cuda')
    ops.bn_bwd_reduce(dout, out, y, saved, sums, 1)
    ops.bn_bwd_apply(dout, out, y, saved, gamma, sums, dy, dres, dgamma, dbeta, 1)
    scale = max(1.0, rows ** 0.5)
    _close(dbeta, b.grad, 2e-2, 2e-2 * scale, 'dbeta')
    _close(dgamma, g.grad, 2e-2, 2e-2 * scale, 'dgamma')
    _close(dres, resf.grad, 1e-2, 1e-2, 'dres', max_bad_frac=1e-3)
    _close(dy, yf.grad, 2e-2, 2e-2, 'bn dy', max_bad_frac=1e-3)
    # plain conv->BN->ReLU unit: the mask is recomputed from y inside the kernels (no `out` read)
    out2 = torch.empty_like(y)
    ops.bn_apply(y, ss, out2, 1)
    yf2 = y.float().requires_grad_(True)
    ref2 = F.relu(F.batch_norm(yf2, None, None, gamma, beta, True, 0.1, 1e-5))
    ref2.backward(dout.float())
    dy2 = torch.empty_like(y)
    ops.bn_bwd_reduce(dout, None, y, saved, sums, 1, scale_shift=ss)
    ops.bn_bwd_apply(dout, None, y, saved, gamma, sums, dy2, None, dgamma, dbeta, 1, scale_shift=ss)
    _close(dy2, yf2.grad, 2e-2, 2e-2, 'bn dy (recomputed mask)', max_bad_frac=1e-3)


def test_maxpool_avgpool():
    ops = _ops()
    n, h, w, c = 3, 14, 14, 64
    x_nchw = _bf(n, c, h, w, seed=17).float().requires_grad_(True)
    x = x_nchw.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    y, am = ops.maxpool3x3s2_fwd(x)
    ref = F.max_pool2d(x_nchw, 3, 2, 1)
    _close(y, ref.permute(0, 2, 3, 1), 0, 0, 'maxpool fwd')
    dy_nchw = _bf(*ref.shape, seed=18).float()
    ref.backward(dy_nchw)
    dx = ops.maxpool3x3s2_bwd(dy_nchw.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), am, h, w)
    _close(dx, x_nchw.grad.permute(0, 2, 3, 1), 1e-2, 1e-2, 'maxpool bwd')
    a = ops.avgpool_fwd(x)
    _close(a, x.float().mean(dim=(1, 2)), 1e-2, 1e-2, 'avgpool fwd')
    da = _bf(n, c, seed=19)
    dxa = ops.avgpool_bwd(da, h, w)
    _close(dxa, (da.float() / (h * w))[:, None, None, :].expand(n, h, w, c), 1e-2, 1e-3, 'avgpool bwd')


def test_colsum_cast_add():
    ops = _ops()
    x = _bf(1000, 768, seed=20)
    out = torch.empty(768, device='cuda')
    ops.colsum(x, out)
    _close(out, x.float().sum(0), 1e-3, 1e-2, 'colsum bf16')
    xf = torch.randn(256, 1000, device='cuda')
    outf = torch.empty(1000, device='cuda')
    ops.colsum(xf, outf)
    _close(outf, xf.sum(0), 1e-4, 1e-4, 'colsum f32')
    _close(ops.cast_bf16(xf), xf.to(torch.bfloat16), 0, 0, 'cast')
    a, b = _bf(64, 128, seed=21), _bf(64, 128, seed=22)
    ref = (a.float() + b.float())
    ops.add_bf16(a, b)
    _close(a, ref, 1e-2, 1e-2, 'add')
