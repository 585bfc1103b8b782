"""RandomResizedCrop / Resize + CenterCrop + flip on the uint8 input edge at 256 x 224^2 (the ImageNet recipes' batch), one
GPU.  Prints one JSON line with the card's name, power limit and maximum SM clock, read in the same run, and:

- the saicv_u8_resample call for the train geometry (RandomResizedCrop(224) + flip draws) and for the eval geometry
  (Resize(256) + CenterCrop(224)), from CUDA events after a warm-up, averaged over several batches' draws;
- the host->device bytes per batch (the packed crops for training, the whole sources for evaluation) against the
  38.5 MB of a 256 x 224^2 uint8 batch;
- the host time per image of Uint8RandomResizedCrop + Uint8RandomHorizontalFlip (draws + crop copy) against the
  reference's Opencv2PIL + TorchRandomResizedCrop + TorchRandomHorizontalFlip (Pillow), on this machine's CPU (model
  printed; one thread).  The reference is imported from what build() installed under oracle/_ref (baseline/ref_import);
  without it that part is skipped.

Source sizes: ImageNet-like (tests/test_resample_input_gpu.imagenet_like_sizes: 70 % of 500 x 375, 375 x 500,
500 x 333, 333 x 500, 400 x 500 or 500 x 500; 30 % 200..1600 wide with an aspect ratio of 0.5..1.5), and all 1600 x 1200.

    python tests/perf_resample_input.py [--iters 50] [--warmup 5] [--batch 256]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from perf_mixup_input import cpu_model  # noqa: E402
from perf_randaugment_input import gpu_card  # noqa: E402
from test_resample_input_gpu import imagenet_like_sizes  # noqa: E402


def _batch(sizes, seed, train):
    from simpleaicv_pytorch_training_examples_b200.classification import common
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed)
    if train:
        tf = [common.Uint8RandomResizedCrop(224), common.Uint8RandomHorizontalFlip(0.5)]
    else:
        tf = [common.Uint8Resize(256), common.Uint8CenterCrop(224)]
    samples = []
    for h, w in sizes:
        s = {'image': rng.randint(0, 256, size=(h, w, 3), dtype=np.uint8), 'label': 0}
        for t in tf:
            s = t(s)
        samples.append(s)
    return common.pack_resample(samples)


def time_resample(sizes, train, iters, warmup, draws=4):
    from simpleaicv_pytorch_training_examples_b200 import ops
    batches = [_batch(sizes, 100 + d, train) for d in range(draws)]
    dev = [(rs.data.cuda(), rs) for rs in batches]
    out = torch.empty(len(sizes), 224, 224, 3, dtype=torch.uint8, device='cuda')
    per = []
    for src, rs in dev:
        for _ in range(warmup):
            ops.u8_resample(src, rs.offsets, rs.geom, out=out)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(iters):
            ops.u8_resample(src, rs.offsets, rs.geom, out=out)
        end.record()
        end.synchronize()
        per.append(start.elapsed_time(end) * 1e3 / iters)
    h2d = float(np.mean([rs.data.numel() for rs in batches]))
    return {'us_per_batch': [round(v, 1) for v in per], 'us_median': round(float(np.median(per)), 1),
            'h2d_bytes_per_batch': int(h2d), 'h2d_vs_uint8_224_batch': round(h2d / (len(sizes) * 224 * 224 * 3), 3)}


def host_time(shape, n=200):
    from simpleaicv_pytorch_training_examples_b200.classification import common
    torch.set_num_threads(1)
    image = np.random.RandomState(0).randint(0, 256, size=shape + (3,)).astype(np.float32)
    rrc, flip = common.Uint8RandomResizedCrop(224), common.Uint8RandomHorizontalFlip(0.5)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    for _ in range(n):
        flip(rrc({'image': image, 'label': 0}))
    ours = (time.perf_counter() - t0) / n * 1e6
    res = {'shape': list(shape), 'uint8_draws_and_crop_us': round(ours, 1)}
    from baseline import ref_import
    if ref_import.available():
        ref = ref_import.module('SimpleAICV.classification.common')
        tf = [ref.Opencv2PIL(), ref.TorchRandomResizedCrop(resize=224), ref.TorchRandomHorizontalFlip(prob=0.5)]
        t0 = time.perf_counter()
        for _ in range(n):
            s = {'image': image, 'label': 0}
            for t in tf:
                s = t(s)
        res['reference_pil_us'] = round((time.perf_counter() - t0) / n * 1e6, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=256)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'measures on the GPU'
    result = {'card': gpu_card(), 'cpu': cpu_model(), 'batch': a.batch}
    imagenet = imagenet_like_sizes(a.batch, 0)
    large = [(1200, 1600)] * a.batch
    result['train_imagenet_like'] = time_resample(imagenet, True, a.iters, a.warmup)
    result['eval_imagenet_like'] = time_resample(imagenet, False, a.iters, a.warmup)
    result['train_1600x1200'] = time_resample(large, True, a.iters, a.warmup)
    result['eval_1600x1200'] = time_resample(large, False, a.iters, a.warmup)
    result['host_per_image'] = [host_time((375, 500)), host_time((1200, 1600), n=50)]
    print(json.dumps(result))


if __name__ == '__main__':
    main()
