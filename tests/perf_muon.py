"""Muon optimizer-step time on the parameter sets of ResNet-50, ViT-B/16 and the DINOv3 ViT-L/16 backbone: FusedMuon
(multi-tensor prep / apply kernels, batched Newton-Schulz GEMMs per shape class) against an eager torch restatement of
the reference's step with bf16 matmuls (a Python loop over the parameters, Newton-Schulz per matrix), the two timed
alternately in the same run with CUDA events.  Reports the Newton-Schulz FLOPs computed from the shapes, the achieved
rate of the whole fused step over them, and the card's name and power limit read in the same run.  No model runs: the
gradients are seeded random tensors.

    python tests/perf_muon.py [--steps 20] [--warmup 3] [--rounds 3] [--out /tmp/perf_muon.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

COEF = (3.4445, -4.7750, 2.0315)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f'unknown ({e})'


def models():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.detection.models.backbones import dinov3vit
    return {
        'resnet50': lambda: backbones.resnet50(num_classes=1000),
        'vit_base_patch16': lambda: backbones.vit_base_patch16(image_size=224, num_classes=1000),
        'dinov3_vit_large_patch16': lambda: dinov3vit.dinov3_vit_large_patch16_backbone(),
    }


def ns_flops(muon_params, steps=5):
    """2 m n m + 2 m m m + 2 m m n per iteration for each matrix viewed [m, n], m <= n."""
    tot = 0
    for p in muon_params:
        r, c = p.shape[0], p.numel() // p.shape[0]
        m, n = min(r, c), max(r, c)
        tot += steps * (4 * m * m * n + 2 * m * m * m)
    return tot


class EagerMuon:
    """The reference's Muon step in eager torch: bf16 Newton-Schulz per matrix, torch elementwise ops."""

    def __init__(self, muon, adamw, lr, wd, momentum=0.95, betas=(0.9, 0.999), eps=1e-8):
        self.muon, self.adamw, self.lr, self.wd, self.mom, self.betas, self.eps = muon, adamw, lr, wd, momentum, betas, eps
        self.buf = [torch.zeros(p.shape[0], p.numel() // p.shape[0], device=p.device) for p in muon]
        self.m1 = [torch.zeros_like(p) for p in adamw]
        self.m2 = [torch.zeros_like(p) for p in adamw]
        self.t = 0

    @staticmethod
    def ns(g, steps=5):
        a, b, c = COEF
        x = g.to(torch.bfloat16)
        if g.size(0) > g.size(1):
            x = x.mT
        x = x / (x.norm() + 1e-7)
        for _ in range(steps):
            m = x @ x.mT
            bm = b * m + c * m @ m
            x = a * x + bm @ x
        if g.size(0) > g.size(1):
            x = x.mT
        return x.float()

    @torch.no_grad()
    def step(self):
        for p, buf in zip(self.muon, self.buf):
            g = p.grad.view(p.shape[0], -1)
            buf.mul_(self.mom).add_(g)
            u = self.ns(g.add(buf, alpha=self.mom))
            p.mul_(1 - self.lr * self.wd).add_(u.view(p.shape), alpha=-self.lr * 0.2 * math.sqrt(max(p.shape[0], p.shape[1])))
        self.t += 1
        b1, b2 = self.betas
        scale = (1 - b1 ** self.t) / (1 - b2 ** self.t) ** 0.5
        for p, m1, m2 in zip(self.adamw, self.m1, self.m2):
            m1.lerp_(p.grad, 1 - b1)
            m2.lerp_(p.grad.square(), 1 - b2)
            p.mul_(1 - self.lr * self.wd).add_(m1 / (self.eps + m2.sqrt()), alpha=-self.lr / scale)


def time_steps(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def run_one(name, ctor, steps, warmup, rounds):
    from simpleaicv_pytorch_training_examples_b200.tools import utils

    class Cfg:
        optimizer = ('Muon', {'lr': 1e-3, 'weight_decay': 0.05})
    model = ctor().cuda()
    opt, _ = utils.build_optimizer(Cfg, model)
    muon, adamw, _ = utils.muon_split(Cfg.optimizer[1], model)
    ref_model = ctor().cuda()
    named = dict(ref_model.named_parameters())
    eager = EagerMuon([named[n] for n, _ in muon], [named[n] for n, _ in adamw], 1e-3, 0.05)
    g = torch.Generator(device='cuda').manual_seed(0)
    for (_, p), q in zip(model.named_parameters(), ref_model.parameters()):
        p.grad = torch.randn(p.shape, device='cuda', generator=g) * 1e-3
        q.grad = p.grad.clone()
    for _ in range(warmup):
        opt.step()
        eager.step()
    torch.cuda.synchronize()
    fused_ms, eager_ms = [], []
    for _ in range(rounds):     # alternate, so that both see the same clocks and neighbours
        fused_ms.append(time_steps(opt.step, steps))
        eager_ms.append(time_steps(eager.step, steps))
    flops = ns_flops([p for _, p in muon])
    f = min(fused_ms)
    return {
        'params': sum(p.numel() for p in model.parameters()), 'muon_matrices': len(muon), 'adamw_tensors': len(adamw),
        'shape_classes': len(opt._classes), 'ns_tflop_per_step': flops / 1e12,
        'fused_step_ms': f, 'fused_step_ms_rounds': fused_ms, 'eager_torch_bf16_step_ms': min(eager_ms),
        'eager_torch_bf16_step_ms_rounds': eager_ms, 'speedup_vs_eager': min(eager_ms) / f,
        'fused_step_ns_tflops': flops / (f * 1e-3) / 1e12,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--models', default='resnet50,vit_base_patch16,dinov3_vit_large_patch16')
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'perf_muon.py measures on the GPU'
    res = {'card': card(), 'torch': torch.__version__, 'steps': a.steps, 'rounds': a.rounds,
           'note': 'fused_step_ns_tflops = Newton-Schulz FLOPs / whole fused step time (prep, NS, apply)'}
    ms = models()
    for name in a.models.split(','):
        res[name] = run_one(name, ms[name], a.steps, a.warmup, a.rounds)
        print(name, json.dumps(res[name]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
