"""ResNet-50 layer-1/2 conv shapes (bs 256): forward with and without the BatchNorm-statistics epilogue, the separate
bn_stats pass, data and weight gradients.  Answers which part of the small-K / small-C launches is epilogue time."""
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


N = 256
for (h, c, k, r) in ((56, 64, 256, 1), (56, 256, 64, 1), (56, 64, 64, 3), (28, 128, 512, 1), (28, 128, 128, 3), (14, 256, 1024, 1)):
    pad = r // 2
    x = torch.randn(N, h, h, c, device='cuda').bfloat16()
    w = torch.randn(k, r * r * c, device='cuda').bfloat16() * 0.05
    cs = ops.make_conv_shape(N, h, h, c, k, r, r, 1, pad)
    y = torch.empty(N, h, h, k, device='cuda', dtype=torch.bfloat16)
    dy = torch.randn(N, h, h, k, device='cuda').bfloat16()
    dx = torch.empty_like(x)
    stats = ops.partial_ws(x.device, 2 * k)
    bytes_io = (x.numel() + y.numel()) * 2
    res = {
        'fprop': timeit(lambda: ops.conv_fprop(x, w, cs, out=y)),
        'fprop + stats epilogue': timeit(lambda: ops.conv_fprop(x, w, cs, out=y, stats=stats)),
        'bn_stats pass alone': timeit(lambda: ops.bn_stats(y)),
        'dgrad': timeit(lambda: ops.conv_dgrad(dy, w, cs, out=dx)),
        'wgrad': timeit(lambda: ops.conv_wgrad(dy, x, cs)),
    }
    for name, us in res.items():
        print(f'conv {r}x{r} c{c} k{k} {h}x{h}: {name:24s} {us:8.1f} us   (x+y once = {bytes_io / 1e6:.0f} MB -> {bytes_io / 3.35e6:.0f} us at the H100 SXM HBM3 peak)')
