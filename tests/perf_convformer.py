"""ConvFormer-S18 training-step throughput on one GPU: the shipped ImageNet config's step (224x224, batch 256,
drop_path_prob 0.2, AdamW lr 2e-3 / wd 5e-2, clip_max_norm 1, OneHotLabelCELoss on mixup-style soft labels), eager and
replayed from one CUDA graph (graph.GraphedTrainStep).  Prints one JSON line with ms/step, images/s, library launches per
step and the card's name and power limit, read in the same run.

    python tests/perf_convformer.py [--steps 20] [--warmup 3] [--batch 256] [--dump-outputs DIR] [--torch-ref]

--dump-outputs DIR writes the last graphed step's loss and a seeded sample of the updated parameters (as bench.py does),
so two builds can be compared on identical seeded inputs.  --torch-ref adds the unmodified reference modules (oracle/_ref,
installed by build(); skipped when absent) under torch.autocast(bf16) with torch.optim.AdamW on the same card.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ADAMW = ('AdamW', {'lr': 2e-3, 'global_weight_decay': False, 'weight_decay': 5e-2, 'no_weight_decay_layer_name_list': []})


def card():
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(',')]
        return {'name': name, 'power_limit': power, 'sm_clock_max': clk}
    except Exception as e:  # pragma: no cover
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'not read ({type(e).__name__})'}


def batch(B, nc=1000):
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, generator=g)
    lab = torch.randint(0, nc, (B,), generator=g)
    oh = torch.nn.functional.one_hot(lab, nc).float() * 0.9 + 0.1 / nc       # label smoothing 0.1, mixup of two images
    return x.cuda(), (0.5 * oh + 0.5 * oh.roll(1, 0)).cuda()


class _Clipped:
    """The optimizer as train_classification drives it with clip_max_norm (tools/scripts.py): clip, then step."""

    def __init__(self, opt, max_norm):
        self.opt, self.max_norm = opt, max_norm

    def step(self):
        self.opt.clip_grad_norm(self.max_norm)
        self.opt.step()

    def zero_grad(self):
        self.opt.zero_grad()

    def sync_hyper(self):
        self.opt.sync_hyper()

    def after_replay(self):
        self.opt.after_replay()


def timed(fn, k):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(k):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / k


def measure_runtime(args, x, y):
    from simpleaicv_pytorch_training_examples_b200 import _lib
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils

    class Cfg:
        optimizer = ADAMW

    torch.manual_seed(0)
    model = backbones.convformer_s18(num_classes=1000, drop_path_prob=0.2).cuda().train()
    crit = losses.OneHotLabelCELoss()
    opt = _Clipped(tutils.build_optimizer(Cfg, model)[0], 1.0)

    def step():
        loss = crit(model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss

    for _ in range(max(3, args.warmup)):
        step()
    l0 = _lib.launch_count()
    eager_ms = timed(step, args.steps)
    launches = (_lib.launch_count() - l0) / args.steps
    graphed = GraphedTrainStep(model, crit, opt, x, y)
    graphed.replay()
    graph_ms = timed(graphed.replay, args.steps)
    if args.dump_outputs:
        import numpy as np
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, 'loss.npy'), graphed.static_loss.detach().double().reshape(-1).cpu().numpy())
        flat = torch.cat([q.detach().float().reshape(-1) for q in model.parameters()]).cpu()
        idx = torch.randint(0, flat.numel(), (min(flat.numel(), 4 << 20),), generator=torch.Generator().manual_seed(0)).sort().values
        np.save(os.path.join(args.dump_outputs, 'params_sample.npy'), flat[idx].numpy())
    rec = {'eager_ms_per_step': eager_ms, 'graphed_ms_per_step': graph_ms, 'images_per_s_eager': args.batch / eager_ms * 1e3,
           'images_per_s_graphed': args.batch / graph_ms * 1e3, 'launches_per_step': launches,
           'last_loss': float(graphed.static_loss), 'peak_mem_gb': torch.cuda.max_memory_allocated() / 2 ** 30}
    del graphed, model, opt
    torch.cuda.empty_cache()
    return rec


def measure_reference(args, x, y):
    from baseline import ref_import
    if not ref_import.available():
        return 'skipped: reference not installed (oracle/_ref)'
    ref_losses = ref_import.module('SimpleAICV.classification.losses')
    torch.manual_seed(0)
    model = ref_import.backbones().convformer_s18(num_classes=1000, drop_path_prob=0.2).cuda().train()
    crit = ref_losses.OneHotLabelCELoss()
    opt = torch.optim.AdamW(model.parameters(), lr=2e-3, weight_decay=5e-2)

    def step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            loss = crit(model(x), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        opt.step()
        opt.zero_grad()

    for _ in range(max(3, args.warmup)):
        step()
    ms = timed(step, args.steps)
    return {'ms_per_step': ms, 'images_per_s': args.batch / ms * 1e3, 'mode': 'eager torch, autocast(bf16), torch.optim.AdamW'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--dump-outputs', default=None, metavar='DIR')
    ap.add_argument('--torch-ref', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_convformer.py needs a CUDA device')
    x, y = batch(args.batch)
    line = {'workload': f'convformer_s18 224x224 bs{args.batch} training step (drop_path 0.2, AdamW, clip_max_norm 1, OneHotLabelCELoss)',
            'card': card(), 'timed_steps': args.steps, 'runtime': measure_runtime(args, x, y)}
    if args.torch_ref:
        line['torch_reference'] = measure_reference(args, x, y)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
