"""RandAugment on the uint8 input edge at 256 x 224^2 (the ImageNet recipes' batch), one GPU.  Prints one JSON line with
the card's name, power limit and maximum SM clock, read in the same run, and:

- the saicv_u8_rand_augment call (stats + apply kernels of both layers) from CUDA events after a warm-up, on records
  drawn with the shipped arguments (magnitude=9, num_layers=2, magnitude_std=0.5), averaged over several batches' draws;
- the host time per image of Uint8RandAugment (draws only) against the reference's RandAugment (PIL), on this machine's
  CPU (model printed; one thread).  The reference is imported from what build() installed under oracle/_ref
  (baseline/ref_import); without it that part is skipped.

    python tests/perf_randaugment_input.py [--iters 50] [--warmup 5] [--batch 256]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from perf_mixup_input import cpu_model  # noqa: E402

MEAN = (0.485, 0.456, 0.406)
RANDAUG = dict(magnitude=9, num_layers=2, resize=224, mean=list(MEAN), integer=True, weight_idx=None, magnitude_std=0.5,
               magnitude_max=None)


def gpu_card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def images(b, seed=0):
    rng = np.random.RandomState(seed)
    coarse = rng.uniform(40, 190, size=(b, 29, 29, 3))
    field = np.repeat(np.repeat(coarse, 8, 1), 8, 2)[:, :224, :224]
    return np.clip(field + rng.normal(0, 12, size=field.shape), 0, 255).astype(np.uint8)


def records(b, count):
    from simpleaicv_pytorch_training_examples_b200.classification import common
    ra = common.Uint8RandAugment(**RANDAUG)
    img = np.zeros((224, 224, 3), np.uint8)
    out = []
    for k in range(count):
        random.seed(k)
        np.random.seed(k)
        s = [ra({'image': img, 'label': 0}) for _ in range(b)]
        out.append(types.SimpleNamespace(
            randaug_ops=torch.from_numpy(np.stack([x['randaug_ops'] for x in s])).pin_memory(),
            randaug_f=torch.from_numpy(np.stack([x['randaug_f'] for x in s])).pin_memory(),
            randaug_affine=torch.from_numpy(np.stack([x['randaug_affine'] for x in s])).pin_memory(),
            randaug_fill=ra.fill))
    return out


def device_time(args):
    from simpleaicv_pytorch_training_examples_b200 import ops
    x0 = torch.from_numpy(images(args.batch)).cuda()
    x = x0.clone()
    scratch = torch.empty_like(x)
    stats = torch.empty(args.batch, 770, dtype=torch.int32, device='cuda')
    recs = records(args.batch, 8)
    for k in range(args.warmup):
        ops.u8_rand_augment(x, recs[k % len(recs)], scratch=scratch, stats=stats)
    torch.cuda.synchronize()
    per = []
    for k in range(args.iters):
        x.copy_(x0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.u8_rand_augment(x, recs[k % len(recs)], scratch=scratch, stats=stats)
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) * 1e3)
    per.sort()
    return {'batch': args.batch, 'iters': args.iters, 'us_median': round(per[len(per) // 2], 1),
            'us_min': round(per[0], 1), 'us_max': round(per[-1], 1)}


def host_time(n=64):
    from PIL import Image
    from baseline import ref_import
    from simpleaicv_pytorch_training_examples_b200.classification import common
    torch.set_num_threads(1)
    imgs = images(n, seed=1)
    ours = common.Uint8RandAugment(**RANDAUG)
    random.seed(0)
    np.random.seed(0)
    t0 = time.perf_counter()
    for _ in range(5):
        for i in range(n):
            ours({'image': imgs[i], 'label': 0})
    out = {'cpu': cpu_model(), 'uint8_randaugment_us_per_image': round((time.perf_counter() - t0) / (5 * n) * 1e6, 1)}
    if not ref_import.available():
        out['reference_randaugment_us_per_image'] = 'skipped: reference not installed'
        return out
    ar = ref_import.module('SimpleAICV.classification.auto_rand_augment')
    ref = ar.RandAugment(**RANDAUG)
    pil = [Image.fromarray(imgs[i]) for i in range(n)]
    random.seed(0)
    np.random.seed(0)
    t0 = time.perf_counter()
    for _ in range(5):
        for i in range(n):
            ref({'image': pil[i], 'label': 0})
    out['reference_randaugment_us_per_image'] = round((time.perf_counter() - t0) / (5 * n) * 1e6, 1)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--iters', type=int, default=50)
    p.add_argument('--warmup', type=int, default=5)
    p.add_argument('--batch', type=int, default=256)
    args = p.parse_args()
    res = {'card': gpu_card(), 'device': device_time(args), 'host_cpu': host_time()}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
