"""Context number (NOT a bench.py arm): the reference's GPU path on this box, i.e. its model code
(restated by oracle/convnets.py, the same torch ops) executed by stock PyTorch CUDA kernels under
autocast(bf16) + autograd + torch.optim.SGD, with the per-step host syncs of
tools/scripts.py:141-270 (isinf/isnan checks, loss == 0 test, .item()): the reference's
own single-GPU throughput on the same box.

    python tests/perf_torch_gpu_baseline.py [--batch 256] [--steps 10] [--channels-last] [--benchmark]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import convnets, vit  # noqa: E402


def run_vit(a):
    """ViT-B/16 (global_pool, soft labels, AdamW) on stock torch kernels under autocast(bf16): the
    reference's unfused attention / MLP ops (vit.py:62-97) through oracle/vit.py's identical op sequence."""
    dev = torch.device('cuda')
    sd = {k: v.to(dev) for k, v in vit.init_state(a.model, 1000, 0).items()}
    for v in sd.values():
        v.requires_grad_(True)
    opt = torch.optim.AdamW([{'params': [v for v in sd.values() if v.ndim > 1], 'weight_decay': 0.05},
                             {'params': [v for v in sd.values() if v.ndim <= 1], 'weight_decay': 0.}], lr=5e-4)
    x = torch.randn(a.batch, 3, 224, 224, device=dev)
    lab = torch.randint(0, 1000, (a.batch,), device=dev)
    y = torch.nn.functional.one_hot(lab, 1000).float() * 0.9 + 1e-4

    def step():
        if torch.any(torch.isinf(x)) or torch.any(torch.isnan(x)):
            return
        with torch.autocast('cuda', dtype=torch.bfloat16):
            out = vit.forward(sd, x, a.model, global_pool=True)
            loss = torch.sum(-y * torch.nn.functional.log_softmax(out.float(), dim=-1), dim=-1).mean()
        if loss == 0. or torch.any(torch.isinf(loss)) or torch.any(torch.isnan(loss)):
            return
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.item()

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(a.steps):
        step()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / a.steps
    print(json.dumps({'what': 'stock torch (reference GPU path) ViT-B/16 bf16 autocast, drop_path 0', 'batch': a.batch,
                      'ms_per_step': ms, 'images_per_sec': a.batch / ms * 1e3, 'torch': torch.__version__}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--benchmark', action='store_true', help='cudnn.benchmark=True (the reference ships False + deterministic)')
    ap.add_argument('--channels-last', action='store_true')
    ap.add_argument('--model', default='resnet50', choices=['resnet50', 'vit_base_patch16'])
    a = ap.parse_args()
    if a.model != 'resnet50':
        return run_vit(a)
    torch.backends.cudnn.benchmark = a.benchmark
    torch.backends.cudnn.deterministic = not a.benchmark  # tools/utils.py:106-107
    dev = torch.device('cuda')
    sd = {k: v.to(dev) for k, v in convnets.init_state('resnet50', 1000, 0).items()}
    names = convnets.param_names(sd)
    if a.channels_last:
        for n in names:
            if sd[n].ndim == 4:
                sd[n] = sd[n].contiguous(memory_format=torch.channels_last)
    for n in names:
        sd[n].requires_grad_(True)
    decay = [sd[n] for n in names if sd[n].ndim > 1]
    nodecay = [sd[n] for n in names if sd[n].ndim <= 1]
    opt = torch.optim.SGD([{'params': decay, 'weight_decay': 1e-4}, {'params': nodecay, 'weight_decay': 0.}], lr=0.1, momentum=0.9)
    x = torch.randn(a.batch, 3, 224, 224, device=dev)
    if a.channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (a.batch,), device=dev)

    def step():
        if torch.any(torch.isinf(x)) or torch.any(torch.isnan(x)):
            return
        with torch.autocast('cuda', dtype=torch.bfloat16):
            out = convnets.forward(sd, x, 'resnet50', training=True)
            loss = torch.nn.functional.cross_entropy(out.float(), y)
        if loss == 0. or torch.any(torch.isinf(loss)) or torch.any(torch.isnan(loss)):
            return
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.item()

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(a.steps):
        step()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / a.steps
    print(json.dumps({'what': 'stock torch (reference GPU path) ResNet-50 bf16 autocast', 'batch': a.batch,
                      'cudnn_benchmark': a.benchmark, 'channels_last': a.channels_last, 'ms_per_step': ms,
                      'images_per_sec': a.batch / ms * 1e3, 'torch': torch.__version__}))


if __name__ == '__main__':
    main()
