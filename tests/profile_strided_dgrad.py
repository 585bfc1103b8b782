"""Per-launch timing of the stride-2 3x3 data gradients of ResNet-50 (bs 256) and of the DETR-R50 body (1024 px, bs 4):
zero_upsample2 + the stride-1 dgrad over the upsampled dy (the fallback) against the phase dgrad on the compact dy.
CUDA events over 20 launches after 3 warm-up launches; prints the card name and power limit read in the same run."""
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402


def timeit(fn, n=20):
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


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi not available'
    return f'{torch.cuda.get_device_name()} ({q})'


print(card())
for (n, h, c) in ((256, 56, 128), (256, 28, 256), (256, 14, 512), (4, 256, 128), (4, 128, 256), (4, 64, 512)):
    k = c
    cs = ops.make_conv_shape(n, h, h, c, k, 3, 3, 2, 1)
    cs1 = ops.make_conv_shape(n, h, h, c, k, 3, 3, 1, 1)
    P = h // 2
    dy = torch.randn(n, P, P, k, device='cuda').bfloat16()
    w = torch.randn(k, 9 * c, device='cuda').bfloat16() * 0.05
    u = torch.empty(n, h, h, k, device='cuda', dtype=torch.bfloat16)
    dx = torch.empty(n, h, h, c, device='cuda', dtype=torch.bfloat16)
    ups = timeit(lambda: ops.zero_upsample2(dy, h, h, out=u))
    old = timeit(lambda: ops.conv_dgrad(u, w, cs1, out=dx))
    new = timeit(lambda: ops.conv_dgrad(dy, w, cs, out=dx))
    issued, useful = 2.0 * n * h * h * k * c * 9, 2.0 * n * P * P * k * c * 9
    print(f'dgrad 3x3/2 n{n} c{c} k{k} {h}x{h}: zero_upsample2 {ups:8.1f} us + stride-1 dgrad {old:8.1f} us '
          f'({issued / old * 1e-6:6.1f} TFLOP/s issued) -> phase dgrad {new:8.1f} us ({useful / new * 1e-6:6.1f} TFLOP/s); '
          f'saves {ups + old - new:8.1f} us')
