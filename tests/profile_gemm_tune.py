"""Sweep of the GEMM engine's launch knobs (tile width : ring stages : staging slices per epilogue half, the
SAICV_GEMM_TUNE override of csrc/capi_gemm.cu) on the epilogue-bound launches of the ViT-B and ResNet-50 steps, next to
the per-thread-load aux path of round 1 (SAICV_GEMM_NO_AUX_TMA).  CUDA events, 10 launches after 3 warm-ups."""
import os
import sys

import torch

sys.path.insert(0, '.')
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402

HBM, TF = 3.35e12, 989e12   # H100 SXM data sheet: HBM3 bandwidth, dense BF16 (700 W)


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n * 1e3


def sweep(name, fn, flops, nbytes, tunes):
    bound = max(flops / TF, nbytes / HBM) * 1e6
    for t in tunes:
        os.environ.pop('SAICV_GEMM_TUNE', None)
        os.environ.pop('SAICV_GEMM_NO_AUX_TMA', None)
        if t == 'legacy':
            os.environ['SAICV_GEMM_NO_AUX_TMA'] = '1'
        elif t != 'default':
            os.environ['SAICV_GEMM_TUNE'] = t
        try:
            us = timeit(fn)
            print(f'{name:58s} {t:10s} {us:8.1f} us   bound {bound:6.1f} us   frac {bound / us:5.2f}', flush=True)
        except RuntimeError as ex:
            print(f'{name:58s} {t:10s} failed: {str(ex)[:80]}', flush=True)
    os.environ.pop('SAICV_GEMM_TUNE', None)
    os.environ.pop('SAICV_GEMM_NO_AUX_TMA', None)


which = sys.argv[1] if len(sys.argv) > 1 else 'all'

if which in ('all', 'vit'):
    M = 50432
    # proj / fc2 forward with the fp32 residual stream
    for N, K in ((768, 768), (768, 3072)):
        x = torch.randn(M, K, device='cuda').bfloat16()
        w = (torch.randn(N, K, device='cuda') * K ** -0.5).bfloat16()
        b = torch.randn(N, device='cuda')
        r = torch.randn(M, N, device='cuda')
        out = torch.empty(M, N, device='cuda')
        fl, by = 2.0 * M * N * K, 2 * (M * K + N * K) + 8 * M * N
        sweep(f'linear_fwd M{M} N{N} K{K} + fp32 resid -> fp32', lambda: ops.linear_fwd(x, w, bias=b, resid=r, out=out, out_f32=True), fl, by,
              ['legacy', 'default', '256:4:1', '256:3:2', '192:4:2', '192:3:3', '128:4:3', '128:5:2'])
        sweep(f'linear_fwd M{M} N{N} K{K} plain -> fp32', lambda: ops.linear_fwd(x, w, bias=b, out=out, out_f32=True), fl, by - 4 * M * N,
              ['default', '256:4:1', '256:3:2', '192:4:2'])
    # fc2 data gradient (reduction 768 -> 3072 wide) with dGELU / plain; fc1 forward with GELU (768 -> 3072)
    dy = torch.randn(M, 768, device='cuda').bfloat16()
    w = (torch.randn(768, 3072, device='cuda') * 768 ** -0.5).bfloat16()
    aux = torch.randn(M, 3072, device='cuda').bfloat16()
    out = torch.empty(M, 3072, device='cuda', dtype=torch.bfloat16)
    fl = 2.0 * M * 768 * 3072
    by = 2 * (M * 768 + 768 * 3072 + M * 3072)
    sweep('linear_dgrad M50432 red768 out3072 plain', lambda: ops.linear_dgrad(dy, w, out=out), fl, by, ['default', '256:4:1', '256:3:2', '192:4:2'])
    sweep('linear_dgrad M50432 red768 out3072 dGELU', lambda: ops.linear_dgrad(dy, w, out=out, gelu_pre=aux), fl, by + 2 * M * 3072,
          ['legacy', 'default', '256:4:1', '256:3:2', '192:4:2', '192:3:3', '128:4:3'])
    w1 = (torch.randn(3072, 768, device='cuda') * 768 ** -0.5).bfloat16()
    b1 = torch.randn(3072, device='cuda')
    sweep('linear_fwd M50432 N3072 K768 bias -> bf16', lambda: ops.linear_fwd(dy, w1, bias=b1, out=out), fl, by, ['default', '256:4:1', '256:3:2', '192:4:2'])

if which in ('all', 'conv'):
    NB_ = 256
    for (h, c, k, r) in ((56, 64, 256, 1), (56, 256, 64, 1), (56, 64, 64, 3), (28, 128, 512, 1), (28, 512, 128, 1), (14, 256, 1024, 1), (14, 1024, 256, 1)):
        pad = r // 2
        x = torch.randn(NB_, h, h, c, device='cuda').bfloat16()
        w = torch.randn(k, r * r * c, device='cuda').bfloat16() * 0.05
        cs = ops.make_conv_shape(NB_, h, h, c, k, r, r, 1, pad)
        y = torch.empty(NB_, h, h, k, device='cuda', dtype=torch.bfloat16)
        dy = torch.randn(NB_, h, h, k, device='cuda').bfloat16()
        dx = torch.empty_like(x)
        add = torch.randn_like(x)
        stats = ops.partial_ws(x.device, 2 * k)
        fl = 2.0 * NB_ * h * h * c * k * r * r
        by = (x.numel() + y.numel()) * 2
        tag = f'conv {r}x{r} c{c} k{k} {h}x{h}'
        tunes = ['default', '0:0:1', '0:3:2', '0:2:3'] if r == 1 else ['default', '0:0:1']
        sweep(f'{tag} fprop', lambda: ops.conv_fprop(x, w, cs, out=y), fl, by, tunes)
        sweep(f'{tag} fprop + stats', lambda: ops.conv_fprop(x, w, cs, out=y, stats=stats), fl, by, tunes)
        sweep(f'{tag} dgrad', lambda: ops.conv_dgrad(dy, w, cs, out=dx), fl, by, tunes)
        sweep(f'{tag} dgrad + add', lambda: ops.conv_dgrad(dy, w, cs, out=dx, add=add), fl, by + x.numel() * 2, ['legacy'] + tunes + ['0:3:3'])
        sweep(f'{tag} wgrad', lambda: ops.conv_wgrad(dy, x, cs), fl, by, ['default', '0:0:1'])
