"""Launches the epilogue-bound GEMM shapes of ResNet-50 layer 1 a few times each, for a profiler capture
(torch.profiler): conv 1x1 c64->k256 56x56 forward without / with the BatchNorm-statistics epilogue and
the c256->k64 data gradient with the shortcut addend (aux operand by TMA)."""
import sys

import torch

sys.path.insert(0, '.')
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402

N, h = 256, 56
x = torch.randn(N, h, h, 64, device='cuda').bfloat16()
w = torch.randn(256, 64, device='cuda').bfloat16() * 0.05
cs = ops.make_conv_shape(N, h, h, 64, 256, 1, 1, 1, 0)
y = torch.empty(N, h, h, 256, device='cuda', dtype=torch.bfloat16)
stats = ops.partial_ws(x.device, 2 * 256)
dy = torch.randn(N, h, h, 256, device='cuda').bfloat16()
dx = torch.empty_like(x)
add = torch.randn_like(x)
for _ in range(2):
    ops.conv_fprop(x, w, cs, out=y)                 # launches 0, 3
    ops.conv_fprop(x, w, cs, out=y, stats=stats)    # launches 1, 4
    ops.conv_dgrad(dy, w, cs, out=dx, add=add)      # launches 2, 5
torch.cuda.synchronize()
print('done')
