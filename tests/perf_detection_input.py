"""DETR and SAM-encoder inputs on the uint8 edge at 1024^2, one GPU.  Prints one JSON line with the card's name, power
limit and maximum SM clock, read in the same run, and per recipe:

- host us per sample of the reference's chain (float32 cv2 transforms + collater share) against the Uint8* chain (draws,
  flip / crop copies, packing; pageable memory, as the reference's collater: DataLoader(pin_memory=True) pins both), on
  this machine's CPU (model printed; one thread).  The reference is imported from what
  build() installed under oracle/_ref; without it that part is "not measured";
- host->device bytes per step: the reference's fp32 image (+ DETR's bool mask) against the packed uint8 sources;
- the saicv_u8_resize_pad call per batch from CUDA events after a warm-up.
Step time with live DataLoader workers is not measured here.

Sources are COCO-like 640 x 480 / 480 x 640 for DETR (half of them translated, as RandomTranslate(0.5) does) and
SA-1B-like 2250 x 1500 for SAM.

    python tests/perf_detection_input.py [--batch 16] [--iters 20] [--warmup 3]
"""
import argparse
import copy
import importlib.util
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from perf_mixup_input import cpu_model  # noqa: E402
from perf_randaugment_input import gpu_card  # noqa: E402

_spec = importlib.util.spec_from_file_location('mk_detection_input', os.path.join(HERE, 'golden', 'make_detection_input_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


def samples(kind, n, seed):
    rng = np.random.RandomState(seed)
    if kind == 'detr':
        return [mk.detr_sample(rng, *((480, 640) if i % 2 else (640, 480)), empty=False) for i in range(n)]
    return [mk.sam_sample(rng, 1500, 2250) for _ in range(n)]


def chains(kind, ref):
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import common as usam
    if kind == 'detr':
        ours = (mk.detr_chain(udet, 1024, 'Uint8'), udet.Uint8DETRDetectionCollater(resize=1024, resize_type='yolo_style', pin_memory=False))
        theirs = None if ref is None else (mk.detr_chain(ref[0], 1024), ref[0].DETRDetectionCollater(resize=1024, resize_type='yolo_style'))
    else:
        ours = (mk.sam_chain(usam, 1024, 'Uint8'), usam.Uint8SAMBatchCollater(resize=1024, pin_memory=False))
        theirs = None if ref is None else (mk.sam_chain(ref[1], 1024), ref[1].SAMBatchCollater(resize=1024))
    return ours, theirs


def host_us(data, chain, seed):
    data = copy.deepcopy(data)
    t0 = time.perf_counter()
    batch, _ = mk.run(data, chain[0], chain[1], seed)
    return (time.perf_counter() - t0) * 1e6 / len(data), batch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    torch.set_num_threads(1)
    import cv2
    cv2.setNumThreads(1)
    from baseline import ref_import
    ref = None
    if ref_import.available():
        ref_import._ensure_path()
        from SimpleAICV.detection import common as rdet
        from SimpleAICV.interactive_segmentation import common as rsam
        ref = (rdet, rsam)
    from simpleaicv_pytorch_training_examples_b200 import ops
    out = {'card': gpu_card(), 'cpu': cpu_model(), 'batch': args.batch, 'step_time_with_workers': 'not measured'}
    for kind in ('detr', 'sam'):
        data = samples(kind, args.batch, 0)
        ours, theirs = chains(kind, ref)
        us_ours, batch = host_us(data, ours, 0)
        rec = {'host_us_per_sample_uint8': round(us_ours, 1)}
        size = 1024
        ref_bytes = args.batch * 3 * size * size * 4 + (args.batch * size * size if kind == 'detr' else 0)
        rec['h2d_bytes_reference_image'] = ref_bytes
        rp = batch['resize_pad']
        rec['h2d_bytes_uint8_sources'] = int(rp.data.numel())
        if theirs is not None:
            rec['host_us_per_sample_reference'] = round(host_us(data, theirs, 0)[0], 1)
        else:
            rec['host_us_per_sample_reference'] = 'not measured'
        src = rp.data.cuda()
        img = torch.empty(args.batch, 3, size, size, device='cuda')
        mask = torch.empty(args.batch, size, size, dtype=torch.bool, device='cuda')
        for _ in range(args.warmup):
            ops.u8_resize_pad(src, rp, out=img, mask=mask)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.iters):
            ops.u8_resize_pad(src, rp, out=img, mask=mask)
        end.record()
        torch.cuda.synchronize()
        rec['kernel_us_per_batch'] = round(start.elapsed_time(end) * 1e3 / args.iters, 1)
        rec['translated'] = int(rp.geom[:, 5].sum())
        out[kind] = rec
    print(json.dumps(out))


if __name__ == '__main__':
    main()
