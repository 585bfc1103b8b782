"""Per-launch time and tensor-core rate of the GEMM engine at the shapes the benchmarks run: forward, data gradient and
weight gradient of the ResNet-50 bs256 3x3 convolutions of all four stages, of the 1x1 pair of each stage's bottleneck,
and of ViT-B/16's four linear layers at 256 x 197 tokens.  CUDA events around a window of at least 0.2 s per row, after
warm-up.  The card's name and power limit are printed with the table: a rate means nothing without them.

    python tests/profile_gemm_shapes.py            (from the repository root, on an H100)
"""
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402

assert torch.cuda.is_available(), 'profile_gemm_shapes.py measures on the GPU: no CUDA device found'

WINDOW_S = 0.25


def _elapsed_ms(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def timeit(fn):
    """Microseconds per launch over a window of >= WINDOW_S seconds (>= 20 launches), after 3 + 5 warm-up launches."""
    for _ in range(3):
        fn()
    per = _elapsed_ms(fn, 5) / 5
    n = max(20, int(WINDOW_S * 1e3 / max(per, 1e-3)) + 1)
    return _elapsed_ms(fn, n) / n * 1e3


def report(name, rows):
    for what, flop, us in rows:
        print(f'{name:34s} {what:6s} {us:9.1f} us {flop / us * 1e-6:8.1f} TFLOP/s', flush=True)


def conv_rows(n, h, c, k, r):
    pad = r // 2
    x = torch.randn(n, h, h, c, device='cuda').bfloat16()
    w = (torch.randn(k, r * r * c, device='cuda') * 0.05).bfloat16()
    dy = torch.randn(n, h, h, k, device='cuda').bfloat16()
    cs = ops.make_conv_shape(n, h, h, c, k, r, r, 1, pad)
    y, dx = torch.empty_like(dy), torch.empty_like(x)
    part = ops.conv_wgrad(dy, x, cs)
    flop = 2.0 * n * h * h * k * r * r * c
    return [('fprop', flop, timeit(lambda: ops.conv_fprop(x, w, cs, out=y))),
            ('dgrad', flop, timeit(lambda: ops.conv_dgrad(dy, w, cs, out=dx))),
            ('wgrad', flop, timeit(lambda: ops.conv_wgrad(dy, x, cs, partial=part)))]


def linear_rows(m, k, n):
    x = torch.randn(m, k, device='cuda').bfloat16()
    w = (torch.randn(n, k, device='cuda') * 0.05).bfloat16()
    dy = torch.randn(m, n, device='cuda').bfloat16()
    y, dx = torch.empty_like(dy), torch.empty_like(x)
    part = ops.linear_wgrad(dy, x)
    flop = 2.0 * m * k * n
    return [('fprop', flop, timeit(lambda: ops.linear_fwd(x, w, out=y))),
            ('dgrad', flop, timeit(lambda: ops.linear_dgrad(dy, w, out=dx))),
            ('wgrad', flop, timeit(lambda: ops.linear_wgrad(dy, x, partial=part)))]


def main():
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f'card: {card[torch.cuda.current_device()] if card else torch.cuda.get_device_name()} (name, power limit)')
    N = 256
    print('--- ResNet-50 bs256, 3x3 stride 1 (long reductions: K = 9c)')
    for h, c in ((56, 64), (28, 128), (14, 256), (7, 512)):
        report(f'conv 3x3 c{c} k{c} {h}x{h}', conv_rows(N, h, c, c, 3))
    print('--- ResNet-50 bs256, the 1x1 pair of each stage')
    for h, c in ((56, 64), (28, 128), (14, 256), (7, 512)):
        report(f'conv 1x1 c{4 * c} k{c} {h}x{h}', conv_rows(N, h, 4 * c, c, 1))
        report(f'conv 1x1 c{c} k{4 * c} {h}x{h}', conv_rows(N, h, c, 4 * c, 1))
    print('--- ViT-B/16 bs256 (M = 256 x 197 tokens)')
    M = 256 * 197
    for k, n in ((768, 2304), (768, 768), (768, 3072), (3072, 768)):
        report(f'linear M{M} K{k} N{n}', linear_rows(M, k, n))


if __name__ == '__main__':
    main()
