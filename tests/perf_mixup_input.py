"""Mixup / CutMix + RandomErasing on the uint8 input edge at 256 x 224^2 (the ViT fine-tuning recipes' batch), one GPU.
Prints one JSON line with the card's name and power limit, read in the same run, and:

- the saicv_u8_mix_erase_norm kernels (image pass + soft labels) from CUDA events after a warm-up, for a Mixup and a
  CutMix batch, and the GB/s they reach against the algorithmic bytes (uint8 pixels in, fp32 NCHW out, the erase noise,
  the labels);
- the host-to-device bytes per batch of both pipelines: uint8 pixels + int64 labels + the noise, against fp32 images +
  fp32 soft labels;
- the host time per batch of both pipelines on this machine's CPU (model and thread count printed): Uint8RandomErasing +
  Uint8MixupCutmixClassificationCollater, against the same draws followed by the fp32 tail the reference computes on the
  host (TorchMeanStdNormalize, erase, stack, permute, mix, soft labels; restated by oracle/mixup.py);
- ViT-B/16 training steps (one CUDA graph per step, OneHotLabelCELoss, AdamW) fed through CudaPrefetcher from pinned
  uint8 batches with their Mixup record, against the same loop fed from pinned fp32 images and soft labels.

    python tests/perf_mixup_input.py [--steps 20] [--warmup 3] [--batch 256]
"""
import argparse
import json
import os
import platform
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from perf_convformer import card, timed  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
ADAMW = ('AdamW', {'lr': 5e-4, 'global_weight_decay': False, 'weight_decay': 5e-2, 'no_weight_decay_layer_name_list': []})


def cpu_model():
    try:
        with open('/proc/cpuinfo') as f:
            for line in f:
                if line.startswith('model name'):
                    return line.split(':', 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or platform.machine() or 'unknown'


def host_batches(args, count, classes=1000):
    """`count` batches of seeded uint8 224^2 images through the shipped erase + Mixup / CutMix draws, one per mode first."""
    from simpleaicv_pytorch_training_examples_b200.classification import common
    rng = np.random.default_rng(0)
    images = rng.integers(0, 256, size=(args.batch, 224, 224, 3), dtype=np.uint8)
    labels = [int(v) for v in rng.integers(0, classes, size=args.batch)]
    erase = common.Uint8RandomErasing(prob=0.25, mode='pixel', max_count=1)
    collate = common.Uint8MixupCutmixClassificationCollater(num_classes=classes, pin_memory=False)
    out, modes, seed = [], set(), 0
    while len(out) < count:
        np.random.seed(seed)
        seed += 1
        t0 = time.perf_counter()
        batch = collate([erase({'image': images[i], 'label': labels[i]}) for i in range(args.batch)])
        dt = time.perf_counter() - t0
        mode = batch['mixup'].mode
        if len(modes) < 2 and mode in modes:
            continue
        modes.add(mode)
        out.append((batch, dt))
    return out


def measure_kernel(args, batches):
    from simpleaicv_pytorch_training_examples_b200 import ops
    from simpleaicv_pytorch_training_examples_b200.classification import common
    res = {}
    for batch, _ in batches[:2]:
        rec = batch['mixup']
        x, y, noise = batch['image'].cuda(), batch['label'].cuda(), rec.noise.cuda()
        out = torch.empty(args.batch, 3, 224, 224, device='cuda')
        soft = torch.empty(args.batch, rec.num_classes, device='cuda')

        def run():
            ops.u8_mix_erase_normalize(x, y, MEAN, STD, rec, noise, out=out, soft=soft)
        for _ in range(10):
            run()
        ms = min(timed(run, 50) for _ in range(3))
        px = args.batch * 224 * 224
        nbytes = px * 3 + px * 3 * 4 + rec.noise.numel() * 4 + args.batch * 8 + args.batch * rec.num_classes * 4
        name = {common.MIX_MIXUP: 'mixup', common.MIX_CUTMIX: 'cutmix'}[rec.mode]
        res[name] = {'us': ms * 1e3, 'algorithmic_bytes': nbytes, 'GB_per_s': nbytes / (ms * 1e-3) / 1e9,
                     'share_of_3350_GBps': nbytes / (ms * 1e-3) / 3.35e12, 'erased_images': int((rec.rects[:, 2] > 0).sum())}
    return res


def measure_host(args, batches):
    from oracle import mixup as omix
    u8, f32 = [], []
    for batch, dt in batches:
        t0 = time.perf_counter()
        omix.apply(batch['image'], batch['label'], batch['mixup'], MEAN, STD)
        f32.append(dt + time.perf_counter() - t0)
        u8.append(dt)
    return {'cpu': cpu_model(), 'cpu_count': os.cpu_count(), 'torch_threads': torch.get_num_threads(), 'uint8_ms_per_batch': 1e3 * float(np.median(u8)),
            'fp32_ms_per_batch': 1e3 * float(np.median(f32)), 'batches': len(batches)}


def measure_e2e(args, batches):
    from simpleaicv_pytorch_training_examples_b200 import ops
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils

    class Cfg:
        optimizer = ADAMW
    u8 = []
    f32 = []
    for batch, _ in batches:
        rec = batch['mixup']
        img, soft = ops.u8_mix_erase_normalize(batch['image'].cuda(), batch['label'].cuda(), MEAN, STD, rec, rec.noise.cuda())
        f32.append({'image': img.cpu().pin_memory(), 'label': soft.cpu().pin_memory()})
        rec.pin_memory()
        u8.append({'image': batch['image'].pin_memory(), 'label': batch['label'].pin_memory(), 'mixup': rec})
    torch.manual_seed(0)
    model = backbones.vit_base_patch16(num_classes=1000).cuda().train()
    crit = losses.OneHotLabelCELoss()
    opt = tutils.build_optimizer(Cfg, model)[0]
    graphed = GraphedTrainStep(model, crit, opt, f32[0]['image'].cuda(), f32[0]['label'].cuda())

    def loop(host, k, normalize):
        for batch in tutils.CudaPrefetcher((host[i % len(host)] for i in range(k)), normalize=normalize):
            graphed(batch['image'], batch['label']).item()
    res = {}
    for name, host, norm in (('uint8_mixup_record', u8, (MEAN, STD)), ('fp32_images_soft_labels', f32, None)) * 2:
        loop(host, args.warmup, norm)
        ms = timed(lambda: loop(host, args.steps, norm), 1) / args.steps
        res.setdefault(name, []).append(ms)
    return {k: {'ms_per_step': min(v), 'images_per_s': args.batch / min(v) * 1e3, 'rounds_ms': v} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--batch', type=int, default=256)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'perf_mixup_input.py measures on the GPU'
    batches = host_batches(args, 4)
    px = args.batch * 224 * 224
    h2d = {'uint8_record': [px * 3 + args.batch * 8 + b['mixup'].noise.numel() * 4 for b, _ in batches],
           'fp32': px * 3 * 4 + args.batch * 1000 * 4}
    line = {'card': card(), 'batch': args.batch, 'image': [224, 224], 'kernel': measure_kernel(args, batches),
            'h2d_bytes_per_batch': h2d, 'host_collate': measure_host(args, batches), 'vit_b16_e2e': measure_e2e(args, batches)}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
