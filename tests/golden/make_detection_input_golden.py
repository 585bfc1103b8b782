"""Generates tests/golden/detection_input_b200.npz by running the REFERENCE input chains of the two 1024^2 recipes, scaled
down, on seeded synthetic samples:

- DETR: RandomHorizontalFlip -> RandomCrop -> RandomTranslate -> DetectionResize(yolo_style, multi_scale) -> Normalize
  -> DETRDetectionCollater (SimpleAICV/detection/common.py), resize 64 (multi-scale sizes 32 and 64);
- SAM: SamResize -> SamRandomHorizontalFlip -> SamNormalize -> SAMBatchCollater
  (SimpleAICV/interactive_segmentation/common.py), resize 64.

Each batch mixes portrait, landscape and exactly-resize sources, and samples without annotations.  Per batch the file
holds the uint8 chain's record (packed sources, offsets, geometry, translations), the reference's image batch computed
with the default cv2 (IPP on) and oracle/detection_input.py's batch, and for DETR both padding masks.  It pins the oracle
and the device kernel without the reference.  The sizes are small so that the file stays small; the GPU tests run 1024^2
batches against the oracle this pins.

    python tests/golden/make_detection_input_golden.py
"""
import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FIXTURE = os.path.join(HERE, 'detection_input_b200.npz')
RESIZE = 64
# (h, w) of the sources of one batch: landscape, portrait, exactly RESIZE on the long side, larger than RESIZE, tiny
DETR_BATCHES = [(0, [(24, 32), (32, 24), (64, 50), (37, 30)]), (1, [(15, 50), (64, 64), (75, 45), (10, 17)]),
                (2, [(48, 36), (28, 70), (32, 32), (17, 9)])]
SAM_BATCHES = [(3, [(24, 32), (32, 24), (64, 48), (75, 45)]), (4, [(50, 15), (64, 64), (20, 21), (9, 65)])]


def source(rng, h, w):
    """Integer-valued float32 [h, w, 3], the dtype the datasets' decode path returns (no -0.0, which a decoded image
    never holds)."""
    coarse = rng.uniform(0, 255, size=((h + 5) // 6 + 1, (w + 5) // 6 + 1, 3))
    field = np.repeat(np.repeat(coarse, 6, 0), 6, 1)[:h, :w]
    return (np.clip(np.round(field + rng.normal(0, 20, size=(h, w, 3))), 0, 255) + 0.0).astype(np.float32)


def detr_sample(rng, h, w, empty):
    k = 0 if empty else int(rng.randint(1, 4))
    lo = rng.uniform(0.05, 0.4, size=(k, 2)) * [w, h]
    hi = lo + rng.uniform(0.2, 0.55, size=(k, 2)) * [w, h]
    annots = np.concatenate([lo, hi, rng.randint(0, 80, size=(k, 1))], 1).astype(np.float32)
    return {'image': source(rng, h, w), 'annots': annots, 'scale': np.array(1.).astype(np.float32),
            'size': np.array([h, w]).astype(np.float32)}


def sam_sample(rng, h, w):
    mask = np.zeros((h, w), np.float32)
    y0, x0 = rng.randint(0, h // 2 + 1), rng.randint(0, w // 2 + 1)
    mask[y0:y0 + h // 2 + 1, x0:x0 + w // 2 + 1] = 1.
    box = np.array([x0, y0, min(w, x0 + w // 2 + 1), min(h, y0 + h // 2 + 1)], np.float32)
    points = np.array([[x0 + 0.5, y0 + 0.5, 1.], [rng.uniform(0, w), rng.uniform(0, h), 0.]], np.float32)
    prompt_box = box + rng.uniform(-2, 2, size=4).astype(np.float32)
    return {'image': source(rng, h, w), 'box': box, 'mask': mask, 'size': np.array([h, w]).astype(np.float32),
            'prompt_point': points, 'prompt_box': prompt_box, 'prompt_mask': mask.copy()}


def detr_samples(seed, shapes):
    rng = np.random.RandomState(40_000 + seed)
    return [detr_sample(rng, h, w, empty=(i == 3 and seed != 1)) for i, (h, w) in enumerate(shapes)]


def sam_samples(seed, shapes):
    rng = np.random.RandomState(40_000 + seed)
    return [sam_sample(rng, h, w) for h, w in shapes]


def detr_chain(mod, resize=RESIZE, prefix=''):
    """The DETR train transforms of module ``mod`` (the reference's or ours, with ``prefix`` 'Uint8')."""
    g = lambda name: getattr(mod, prefix + name)     # noqa: E731
    return [g('RandomHorizontalFlip')(prob=0.5), g('RandomCrop')(prob=0.5), g('RandomTranslate')(prob=0.5),
            g('DetectionResize')(resize=resize, stride=32, resize_type='yolo_style', multi_scale=True,
                                 multi_scale_range=[0.8, 1.0]), g('Normalize')()]


def sam_chain(mod, resize=RESIZE, prefix=''):
    g = lambda name: getattr(mod, prefix + name)     # noqa: E731
    return [g('SamResize')(resize=resize), g('SamRandomHorizontalFlip')(prob=0.5),
            g('SamNormalize')(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375])]


def run(samples, transforms, collater, seed):
    """Collated batch of deep copies of ``samples`` through ``transforms`` from np.random.seed(seed), and np.random's
    state after it."""
    np.random.seed(seed)
    out = []
    for s in copy.deepcopy(samples):
        for t in transforms:
            s = t(s)
        out.append(s)
    return collater(out), np.random.get_state()


def oracle_batch(rp):
    """oracle/detection_input.py's (image, mask) for a ResizePadBatch."""
    from oracle import detection_input as od
    data, geom, shift = rp.data.numpy(), rp.geom.numpy(), rp.shift.numpy()
    images = []
    for b, off in enumerate(rp.offsets.numpy()):
        h, w, oh, ow, _, tr = (int(v) for v in geom[b])
        src = data[off:off + h * w * 3].reshape(h, w, 3)
        images.append(od.resized(src, oh, ow, tuple(shift[b]) if tr else None))
    return od.write_batch(images, rp.size, rp.mean, rp.std, flips=geom[:, 4], with_mask=True)


def main():
    from baseline import ref_import
    ref_import._ensure_path()
    from SimpleAICV.detection import common as rdet
    from SimpleAICV.interactive_segmentation import common as rsam
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import common as usam
    arrays = {}
    for kind, batches in (('detr', DETR_BATCHES), ('sam', SAM_BATCHES)):
        for seed, shapes in batches:
            if kind == 'detr':
                samples = detr_samples(seed, shapes)
                ref, _ = run(samples, detr_chain(rdet), rdet.DETRDetectionCollater(resize=RESIZE, resize_type='yolo_style'), seed)
                ours, _ = run(samples, detr_chain(udet, prefix='Uint8'),
                              udet.Uint8DETRDetectionCollater(resize=RESIZE, resize_type='yolo_style', pin_memory=False), seed)
            else:
                samples = sam_samples(seed, shapes)
                ref, _ = run(samples, sam_chain(rsam), rsam.SAMBatchCollater(resize=RESIZE), seed)
                ours, _ = run(samples, sam_chain(usam, prefix='Uint8'), usam.Uint8SAMBatchCollater(resize=RESIZE, pin_memory=False), seed)
            rp = ours['resize_pad']
            image, mask = oracle_batch(rp)
            key = f'{kind}{seed}_'
            arrays.update({key + 'data': rp.data.numpy(), key + 'offsets': rp.offsets.numpy(), key + 'geom': rp.geom.numpy(),
                           key + 'shift': rp.shift.numpy(), key + 'oracle_image': image, key + 'oracle_mask': mask,
                           key + 'ref_image': ref['image'].numpy()})
            if kind == 'detr':
                arrays[key + 'ref_mask'] = ref['mask'].numpy()
    np.savez_compressed(FIXTURE, **arrays)
    print(FIXTURE, os.path.getsize(FIXTURE), 'bytes')


if __name__ == '__main__':
    main()
