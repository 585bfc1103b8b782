"""Cost of the GEMM epilogue variants at the ViT-B fc2 data-gradient shape (M 50432, reduction 768, output 3072) and
the SAM-H one (M 32768, 1280 -> 5120): plain, + dGELU(aux), * (aux > 0), + aux."""
import sys

import torch

sys.path.insert(0, '.')
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402


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


for M, N, K in ((50432, 768, 3072), (32768, 1280, 5120)):
    dy = torch.randn(M, N, device='cuda').bfloat16()
    w = torch.randn(N, K, device='cuda').bfloat16()
    aux = torch.randn(M, K, device='cuda').bfloat16()
    out = torch.empty(M, K, device='cuda', dtype=torch.bfloat16)
    fl = 2.0 * M * N * K
    res = {
        'plain': timeit(lambda: ops.linear_dgrad(dy, w, out=out)),
        'dgelu epilogue': timeit(lambda: ops.linear_dgrad(dy, w, out=out, gelu_pre=aux)),
        'drelu epilogue': timeit(lambda: ops.linear_dgrad(dy, w, out=out, relu_out=aux)),
        'add epilogue': timeit(lambda: ops.linear_dgrad(dy, w, out=out, add=aux)),
    }
    for k, us in res.items():
        print(f'dgrad M{M} N{N} K{K} {k:26s} {us:8.1f} us  {fl / us / 1e6:7.0f} TFLOP/s')
