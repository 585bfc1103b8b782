"""Generates tests/golden/mixup_erase_b6.ptu by running the REFERENCE train tail of the ImageNet recipes with soft labels on
seeded uint8 batches of 6 non-square images:

- TorchMeanStdNormalize + RandomErasing(prob=0.25, mode='pixel', max_count=1) per sample
  (SimpleAICV/classification/common.py:228-248,560-642);
- MixupCutmixClassificationCollater with the shipped arguments (mixupcutmixclassificationcollator.py:99-284).

Each case's np.random seed is the first one whose draws give the case (found with the uint8 counterparts in
classification/common.py, which make the same draws): Mixup with an erased partner, CutMix boxes clipped at the top-left
and at the bottom-right borders, an empty CutMix box (lambda corrected to 1), an erase rectangle overlapping the CutMix box
and Mixup at an image size whose pixel count is not a multiple of 4, and a batch the mixup_cutmix_prob gate leaves unmixed.
The fixture holds the uint8 inputs, labels, seeds and the reference's fp32 images and soft labels.  The file is not a .pt:
tests/test_oracle_golden.py loads every *.pt as a network fixture.

    python tests/golden/make_mixup_golden.py
"""
import contextlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

FIXTURE = os.path.join(HERE, 'mixup_erase_b6.ptu')
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
NUM_CLASSES = 10
ERASE = dict(prob=0.25, mode='pixel', max_count=1)
COLLATE = dict(use_mixup=True, mixup_alpha=0.8, cutmix_alpha=1.0, cutmix_minmax=None, mixup_cutmix_prob=1.0,
               switch_to_cutmix_prob=0.5, mode='batch', correct_lam=True, label_smoothing=0.1, num_classes=NUM_CLASSES)
DRAWS = ('uniform', 'randint', 'normal', 'rand', 'beta')


def make_inputs(seed, b, h, w, num_classes=NUM_CLASSES):
    """uint8 [b, h, w, 3] images and int labels from their own generator (the global np.random state is untouched)."""
    rng = np.random.default_rng(10_000 + seed)
    return rng.integers(0, 256, size=(b, h, w, 3), dtype=np.uint8), [int(v) for v in rng.integers(0, num_classes, size=b)]


@contextlib.contextmanager
def draw_log():
    """Records (name, result) of every np.random.<uniform|randint|normal|rand|beta> call made inside the block."""
    log, saved = [], {n: getattr(np.random, n) for n in DRAWS}

    def wrap(name, fn):
        def call(*args, **kwargs):
            r = fn(*args, **kwargs)
            log.append((name, np.array(r, copy=True)))
            return r
        return call
    for n, fn in saved.items():
        setattr(np.random, n, wrap(n, fn))
    try:
        yield log
    finally:
        for n, fn in saved.items():
            setattr(np.random, n, fn)


def reference_batch(images, labels, seed, **collate):
    """The reference's batch for these inputs from np.random.seed(seed), and the np.random state after it."""
    from baseline import ref_import
    ref = ref_import.module('SimpleAICV.classification.common')
    np.random.seed(seed)
    norm, erase = ref.TorchMeanStdNormalize(mean=list(MEAN), std=list(STD)), ref.RandomErasing(**ERASE)
    samples = [erase(norm({'image': images[i].copy(), 'label': labels[i]})) for i in range(len(labels))]
    batch = ref.MixupCutmixClassificationCollater(**{**COLLATE, **collate})(samples)
    return batch, np.random.get_state()


def uint8_batch(images, labels, seed, **collate):
    """The same from Uint8RandomErasing + Uint8MixupCutmixClassificationCollater (host tensors, not pinned)."""
    from simpleaicv_pytorch_training_examples_b200.classification import common
    np.random.seed(seed)
    erase = common.Uint8RandomErasing(**ERASE)
    samples = [erase({'image': images[i].copy(), 'label': labels[i]}) for i in range(len(labels))]
    batch = common.Uint8MixupCutmixClassificationCollater(**{**COLLATE, **collate}, pin_memory=False)(samples)
    return batch, np.random.get_state()


def _overlaps(rect, box):
    top, left, h, w = (int(v) for v in rect)
    yl, yh, xl, xh = box
    return h > 0 and w > 0 and top < yh and yl < top + h and left < xh and xl < left + w


def _clipped(log, rec, h, w):
    """(top, bottom, left, right) clipping of the CutMix box, from the beta draw and the centre draws."""
    lam_raw = float(log[-3][1])
    cy, cx = int(log[-2][1]), int(log[-1][1])
    ratio = np.sqrt(1 - lam_raw)
    ch, cw = int(h * ratio), int(w * ratio)
    return cy - ch // 2 < 0, cy + ch // 2 > h, cx - cw // 2 < 0, cx + cw // 2 > w


def _case_holds(name, rec, log, h, w):
    from simpleaicv_pytorch_training_examples_b200.classification.common import MIX_CUTMIX, MIX_MIXUP, MIX_NONE
    erased = any(int(r[2]) > 0 for r in rec.rects)
    if name in ('mixup_erased_partner', 'mixup_odd_size'):
        return rec.mode == MIX_MIXUP and erased
    if name == 'no_mix':
        return rec.mode == MIX_NONE and erased
    if rec.mode != MIX_CUTMIX:
        return False
    yl, yh, xl, xh = rec.box
    area = (yh - yl) * (xh - xl)
    if name == 'cutmix_empty_box':
        return area == 0 and rec.lam == 1.
    top, bottom, left, right = _clipped(log, rec, h, w)
    if name == 'cutmix_clip_top_left':
        return area > 0 and top and left and not bottom and not right
    if name == 'cutmix_clip_bottom_right':
        return area > 0 and bottom and right and not top and not left
    if name == 'cutmix_erase_in_box':
        return area > 0 and any(_overlaps(r, rec.box) for r in rec.rects)
    raise KeyError(name)


# name, (h, w), collater overrides
CASES = [('mixup_erased_partner', (10, 14), {}),
         ('cutmix_clip_top_left', (10, 14), {}),
         ('cutmix_clip_bottom_right', (10, 14), {}),
         ('cutmix_empty_box', (10, 14), {}),
         ('cutmix_erase_in_box', (10, 14), {}),
         ('mixup_odd_size', (9, 13), {}),
         ('no_mix', (10, 14), {'mixup_cutmix_prob': 0.5})]


def find_seed(name, hw, collate, b=6):
    for seed in range(100_000):
        images, labels = make_inputs(seed, b, *hw)
        with draw_log() as log:
            batch, _ = uint8_batch(images, labels, seed, **collate)
        if _case_holds(name, batch['mixup'], log, *hw):
            return seed
    raise RuntimeError(f'no seed gives {name}')


def main():
    cases = []
    for name, hw, collate in CASES:
        seed = find_seed(name, hw, collate)
        images, labels = make_inputs(seed, 6, *hw)
        batch, _ = reference_batch(images, labels, seed, **collate)
        cases.append({'name': name, 'seed': seed, 'collate': collate, 'images': torch.from_numpy(images),
                      'labels': torch.tensor(labels, dtype=torch.int64),
                      'image': batch['image'].contiguous().clone(), 'label': batch['label'].clone()})
        print(name, 'seed', seed)
    torch.save({'mean': MEAN, 'std': STD, 'erase': ERASE, 'collate': COLLATE, 'cases': cases}, FIXTURE)
    print('wrote', FIXTURE, os.path.getsize(FIXTURE), 'bytes')


if __name__ == '__main__':
    main()
