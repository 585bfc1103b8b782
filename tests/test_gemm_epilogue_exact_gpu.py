"""The fused GEMM epilogue, bit for bit: each output equals the documented elementwise formula applied in torch to the
fp32 accumulator of the same product.

The accumulator comes from the same engine with no epilogue and fp32 output, on the same operands, operand layouts and
tile width (every output column is one wgmma dot product per k16 step in k-block order whatever the epilogue, see
test_gemm_conformance_gpu.py).  The formulas, in the order the epilogue applies them, one fp32 rounding per operation:

    y = acc (+ bias) -> max(y, 0) -> (+ fp32 residual) -> (+ bf16 addend | y if relu_out > 0 else 0) -> (* mask bit)
    NS:  y = fma(beta, aux, alpha * acc)

and a bf16 output is the round-to-nearest-even of the fp32 result.  Every variant of the kernel and both tile widths
run on ragged shapes (M and N not multiples of the tile).  dGELU and the drop-path row scale are left to the tolerance
checks of test_gemm_conformance_gpu.py: their factors involve MUFU approximations and possible FMA contraction.
"""
import ctypes

import pytest
import torch

from conformance import call, randn, rne_bf16, same

from simpleaicv_pytorch_training_examples_b200 import ops

BNS = (64, 128)
M, RED, N = 1000, 200, 200          # rows, reduction, output columns of the linear cases


def _bf(*shape, scale=1.0, seed=0):
    return randn(*shape, scale=scale, seed=seed).to(torch.bfloat16)


def _bf16_of(acc32):
    """fp32 tensor -> its bf16 rounding (ties to even), as bf16."""
    return rne_bf16(acc32.double()).to(torch.bfloat16)


def _expect(env, monkeypatch, bn):
    monkeypatch.setenv('SAICV_GEMM_TUNE', f'{bn}:0:0')
    for k in ('SAICV_GEMM_FULL_VARIANT', 'SAICV_GEMM_NO_AUX_TMA'):
        monkeypatch.delenv(k, raising=False)
    if env:
        monkeypatch.setenv(env, '1')


# (case, override): the override moves the same launch to VAR_FULL (run-time flags) or to per-thread aux loads
LINEAR_CASES = [
    ('fwd_bias_relu_bf16', None),                      # VAR_PLAIN_BF16
    ('fwd_bias_relu_bf16', 'SAICV_GEMM_FULL_VARIANT'),
    ('fwd_bias_f32', None),                            # VAR_PLAIN_F32
    ('fwd_bias_f32', 'SAICV_GEMM_FULL_VARIANT'),
    ('fwd_stats_bf16', None),                          # VAR_STATS_BF16
    ('fwd_bias_resid_f32', None),                      # VAR_AUX, fp32 aux by TMA
    ('fwd_bias_resid_f32', 'SAICV_GEMM_FULL_VARIANT'),
    ('fwd_bias_resid_f32', 'SAICV_GEMM_NO_AUX_TMA'),   # VAR_FULL, per-thread loads
    ('dgrad_add_bf16', None),                          # VAR_AUX, bf16 aux by TMA
    ('dgrad_add_bf16', 'SAICV_GEMM_FULL_VARIANT'),
    ('dgrad_add_bf16', 'SAICV_GEMM_NO_AUX_TMA'),
    ('dgrad_relu_out_bf16', None),
    ('dgrad_relu_out_bf16', 'SAICV_GEMM_NO_AUX_TMA'),
    ('dgrad_resid_f32', None),
    ('dgrad_resid_f32', 'SAICV_GEMM_NO_AUX_TMA'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
@pytest.mark.parametrize('case,env', LINEAR_CASES)
def test_linear_epilogue_is_formula_of_accumulator(case, env, bn, monkeypatch):
    x, w = _bf(M, RED, seed=1), _bf(N, RED, scale=RED ** -0.5, seed=2)       # forward: y = x w^T
    dy, wd = _bf(M, RED, seed=3), _bf(RED, N, scale=RED ** -0.5, seed=4)     # data gradient: dx = dy wd
    bias = randn(N, scale=0.5, seed=5)
    resid = randn(M, N, seed=6)
    aux = _bf(M, N, seed=7)
    _expect(None, monkeypatch, bn)
    if case.startswith('fwd'):
        acc = ops.linear_fwd(x, w, out_f32=True)
    else:
        acc = ops.linear_dgrad(dy, wd, out_f32=True)
    _expect(env, monkeypatch, bn)
    if case == 'fwd_bias_relu_bf16':
        got, want = ops.linear_fwd(x, w, bias=bias, flags=ops.EPI_RELU), _bf16_of((acc + bias).clamp_min(0))
    elif case == 'fwd_bias_f32':
        got, want = ops.linear_fwd(x, w, bias=bias, out_f32=True), acc + bias
    elif case == 'fwd_stats_bf16':
        ws = torch.zeros(ops.gemm_stats_rows(M, N), 2, N, device='cuda')
        got, want = ops.linear_fwd(x, w, stats=ws), _bf16_of(acc)
    elif case == 'fwd_bias_resid_f32':
        got, want = ops.linear_fwd(x, w, bias=bias, resid=resid, out_f32=True), (acc + bias) + resid
    elif case == 'dgrad_add_bf16':
        got, want = ops.linear_dgrad(dy, wd, add=aux), _bf16_of(acc + aux.float())
    elif case == 'dgrad_relu_out_bf16':
        got, want = ops.linear_dgrad(dy, wd, relu_out=aux), _bf16_of(torch.where(aux.float() > 0, acc, torch.zeros_like(acc)))
    else:
        got, want = ops.linear_dgrad(dy, wd, resid=resid, out_f32=True), acc + resid
    same(f'{case} BN={bn} {env or "default"}', got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
@pytest.mark.parametrize('mask', [False, True])
def test_conv_dgrad_add_mask_epilogue_is_formula_of_accumulator(mask, bn, monkeypatch):
    """1x1 stride-1 data gradient + shortcut gradient (* 1-bit ReLU mask): VAR_AUX.  Its accumulator is the linear data
    gradient dy[pixels, k] w[k, c] (same operand layouts: A K-major, B MN-major)."""
    n, h, w, c, k = 4, 29, 29, 192, 128
    dy = _bf(n, h, w, k, seed=8)
    wb = _bf(k, c, scale=k ** -0.5, seed=9)
    add = _bf(n, h, w, c, seed=10)
    bits = torch.randint(-2 ** 31, 2 ** 31, (n * h * w, c // 32), device='cuda', dtype=torch.int32,
                         generator=torch.Generator(device='cuda').manual_seed(11)) if mask else None
    cs = ops.make_conv_shape(n, h, w, c, k, 1, 1, 1, 0)
    _expect(None, monkeypatch, bn)
    acc = ops.linear_dgrad(dy.view(-1, k), wb, out_f32=True)
    got = ops.conv_dgrad(dy, wb, cs, add=add, mask_bits=bits)
    y = acc + add.view(-1, c).float()
    if mask:
        b = bits.view(torch.uint8).long()          # little-endian: byte j of a word holds channels 8j .. 8j+7 of it
        keep = ((b.unsqueeze(-1) >> torch.arange(8, device='cuda')) & 1).reshape(-1, c).float()
        y = y * keep
    same(f'conv_dgrad add{"+mask" if mask else ""} BN={bn}', got.view(-1, c), _bf16_of(y))


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
def test_phase_dgrad_store_is_rounded_accumulator(bn, monkeypatch):
    """3x3 / stride-2 data gradient by output phase (VAR_PHASE_BF16): each dx pixel is the bf16 rounding of its
    accumulator.  That accumulator is the stride-1 data gradient over the zero-upsampled dy, in the same reduction order
    (taps mirrored, then channels): here as a linear data gradient over an explicit im2col matrix."""
    n, h, w, c, k = 10, 30, 30, 192, 64
    dy = _bf(n, h // 2, w // 2, k, seed=12)
    wb = _bf(k, 9 * c, scale=(9 * c) ** -0.5, seed=13)          # [k][tap * c + ch], tap = r * 3 + s
    cs = ops.make_conv_shape(n, h, w, c, k, 3, 3, 2, 1)
    assert ops.phase_dgrad_ok(cs)
    up = torch.zeros(n, h + 2, w + 2, k, device='cuda', dtype=torch.bfloat16)
    up[:, 1:h + 1:2, 1:w + 1:2] = dy                            # zero-upsampled dy, padded by 1
    a = torch.cat([up[:, r:r + h, s:s + w] for r in range(3) for s in range(3)], dim=-1).view(-1, 9 * k)
    b = torch.cat([wb[:, (8 - t) * c:(9 - t) * c] for t in range(9)], dim=0).contiguous()   # [tap * k + kk][ch]
    _expect(None, monkeypatch, bn)
    acc = ops.linear_dgrad(a.contiguous(), b, out_f32=True)
    got = ops.conv_dgrad(dy, wb, cs)
    same(f'phase dgrad BN={bn}', got.view(-1, c), _bf16_of(acc))


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
def test_ns_axpby_epilogue_is_formula_of_accumulator(bn, monkeypatch):
    """Newton-Schulz product out = alpha x y + beta y (VAR_NS, bf16 aux by TMA) over a batch of two matrices.  The
    accumulator x y is the linear data gradient of x [m, m] and y [m, n] (A K-major, B MN-major)."""
    batch, m, n = 2, 200, 328
    alpha, beta = -4.7750, 2.0315
    x = _bf(batch, m, m, scale=m ** -0.5, seed=14)
    y = _bf(batch, m, n, seed=15)
    _expect(None, monkeypatch, bn)
    acc = torch.stack([ops.linear_dgrad(x[i], y[i], out_f32=True) for i in range(batch)])
    out = torch.empty(batch, m, n, device='cuda', dtype=torch.bfloat16)
    call('saicv_ns_gemm', 2, x, y, out, batch, m, n, ctypes.c_float(alpha), ctypes.c_float(beta))
    a32 = torch.tensor(alpha, dtype=torch.float32).item()
    b32 = torch.tensor(beta, dtype=torch.float32).item()
    t = (acc * a32).double()                                    # alpha * acc, rounded to fp32
    want = (y.double() * b32 + t).float()                       # the fma, one fp32 rounding (exact in float64 here)
    same(f'ns axpby BN={bn}', out, _bf16_of(want))
