"""Attention kernels at the ViT-B/16 bs256 shape (and optionally others) for ncu / quick timing."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from simpleaicv_pytorch_training_examples_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--b', type=int, default=256)
ap.add_argument('--l', type=int, default=197)
ap.add_argument('--h', type=int, default=12)
ap.add_argument('--d', type=int, default=64)
ap.add_argument('--iters', type=int, default=3)
a = ap.parse_args()
g = torch.Generator(device='cuda').manual_seed(0)
qkv = torch.randn(a.b * a.l, 3 * a.h * a.d, device='cuda', generator=g).to(torch.bfloat16)
dout = torch.randn(a.b * a.l, a.h * a.d, device='cuda', generator=g).to(torch.bfloat16)
out, dqkv = torch.empty_like(dout), torch.empty_like(qkv)
q, k, v, o, do, dq, dk, dv = (view for x in (qkv, out, dout, dqkv) for view in ops.head_views(x, a.b, a.l, a.h, a.d))
scale = a.d ** -0.5
for _ in range(2):
    _, lse = ops.attn_fwd(q, k, v, scale, out=o)
    ops.attn_bwd(q, k, v, o, lse, do, scale, dq, dk, dv)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
ev[0].record()
for _ in range(a.iters):
    _, lse = ops.attn_fwd(q, k, v, scale, out=o)
ev[1].record()
for _ in range(a.iters):
    ops.attn_bwd(q, k, v, o, lse, do, scale, dq, dk, dv)
ev[2].record()
torch.cuda.synchronize()
print(f'attention B{a.b} L{a.l} H{a.h} D{a.d}: fwd {ev[0].elapsed_time(ev[1]) / a.iters * 1e3:.1f} us, '
      f'bwd {ev[1].elapsed_time(ev[2]) / a.iters * 1e3:.1f} us')
