"""Generates tests/golden/randaug_b200.ptr by running the REFERENCE RandAugment (SimpleAICV/classification/
auto_rand_augment.py:646-690, the shipped arguments magnitude=9, num_layers=2, magnitude_std=0.5, integer=True,
ImageNet mean) on seeded uint8 images through Pillow:

- 'seeds': whole RandAugment calls on 224 x 224 images from random.seed(s) / np.random.seed(s), with the draws
  classification.common.Uint8RandAugment records for them;
- 'ops': every op of the increasing set forced one at a time on a 13 x 17 image, at magnitudes 0, 9 and 10, both signs
  of the negate draw and both resamples of the geometric ops.  The reference's AugmentOp and Uint8RandAugment's layer
  draw read the same scripted values from a stand-in for the ``random`` module.

The fixture holds the records and the reference's uint8 outputs; the inputs are regenerated from their seeds by
``make_image`` (np.random.RandomState, whose stream numpy keeps fixed).  The file is not a .pt: tests/test_oracle_golden.py
loads every *.pt as a network fixture.

    python tests/golden/make_randaug_golden.py
"""
import contextlib
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

FIXTURE = os.path.join(HERE, 'randaug_b200.ptr')
MEAN = (0.485, 0.456, 0.406)
RANDAUG = dict(magnitude=9, num_layers=2, resize=224, mean=list(MEAN), integer=True, weight_idx=None, magnitude_std=0.5,
               magnitude_max=None)
SEEDS = (18, 99, 21)      # Sharpness + bicubic Rotate, Equalize + bicubic Rotate, Brightness + Contrast
OP_SIZE = (13, 17)
MAGNITUDES = (0., 9., 10.)


def make_image(seed, h, w):
    """uint8 [h, w, 3]: a smooth random field in a narrow range plus noise, so that AutoContrast and Equalize move it."""
    rng = np.random.RandomState(20_000 + seed)
    coarse = rng.uniform(40, 190, size=((h + 7) // 8 + 1, (w + 7) // 8 + 1, 3))
    field = np.repeat(np.repeat(coarse, 8, 0), 8, 1)[:h, :w]
    return np.clip(field + rng.normal(0, 12, size=(h, w, 3)), 0, 255).astype(np.uint8)


def record(sample):
    return sample['randaug_ops'], sample['randaug_f'], sample['randaug_affine']


def reference_sample(image, seed):
    """The reference's RandAugment output for ``image`` from random.seed(seed) / np.random.seed(seed), and the two
    generators' states after it."""
    from PIL import Image
    from baseline import ref_import
    ar = ref_import.module('SimpleAICV.classification.auto_rand_augment')
    random.seed(seed)
    np.random.seed(seed)
    out = ar.RandAugment(**RANDAUG)({'image': Image.fromarray(image), 'label': 0})['image']
    return np.asarray(out), (random.getstate(), np.random.get_state())


def uint8_sample(image, seed, **kw):
    """Uint8RandAugment's sample for the same, and the states after it."""
    from simpleaicv_pytorch_training_examples_b200.classification import common
    random.seed(seed)
    np.random.seed(seed)
    sample = common.Uint8RandAugment(**{**RANDAUG, **kw})({'image': image.copy(), 'label': 0})
    return sample, (random.getstate(), np.random.get_state())


class Scripted:
    """Stands in for the ``random`` module: random() -> 0.0 (the op runs; no negation) or 1.0 on the negate draw when
    ``negate``, gauss() -> ``magnitude``, choice() -> ``resample``."""

    def __init__(self, magnitude, negate, resample):
        self.magnitude, self.negate, self.resample, self.calls = magnitude, negate, resample, 0

    def random(self):
        self.calls += 1
        return 1.0 if self.calls > 1 and self.negate else 0.0

    def gauss(self, mu, sigma):
        return self.magnitude

    def choice(self, seq):
        assert self.resample in seq
        return self.resample


@contextlib.contextmanager
def scripted(module, draws):
    saved = module.random
    module.random = draws
    try:
        yield
    finally:
        module.random = saved


def forced_layer(op, magnitude, negate, resample, h, w):
    """Uint8RandAugment's layer draw for op with scripted draws -> (ops int32 [1, 4], f float32 [1], affine f64 [1, 6])."""
    from simpleaicv_pytorch_training_examples_b200.classification import common
    ra = common.Uint8RandAugment(**RANDAUG)
    with scripted(common, Scripted(magnitude, negate, resample)):
        o, rs, ip, f, coeffs = ra._layer(op, w, h)
    return (np.array([[o, rs, ip, 0]], np.int32), np.array([f], np.float32), np.array([coeffs], np.float64))


def reference_op(image, op, magnitude, negate, resample):
    """The reference AugmentOp(name, prob=0.5, magnitude, hparams of RandAugment) on ``image`` with scripted draws."""
    from PIL import Image
    from baseline import ref_import
    from simpleaicv_pytorch_training_examples_b200.classification import common
    ar = ref_import.module('SimpleAICV.classification.auto_rand_augment')
    aug = ar.RandAugment(**RANDAUG).ops[op]
    assert aug.name == common.RANDAUG_OPS[op]
    with scripted(ar, Scripted(magnitude, negate, resample)):
        return np.asarray(aug(Image.fromarray(image)))


def op_cases():
    """(op, magnitude, negate, resample) for every forced-op case."""
    from simpleaicv_pytorch_training_examples_b200.classification import common
    geometric = {'Rotate', 'ShearX', 'ShearY', 'TranslateXRel', 'TranslateYRel'}
    signed = geometric | {n for n in common.RANDAUG_OPS if n.endswith('Increasing') and not n.startswith(('Posterize',
                                                                                                           'Solarize'))}
    cases = []
    for op, name in enumerate(common.RANDAUG_OPS):
        for m in MAGNITUDES:
            for negate in ((False, True) if name in signed else (False,)):
                for rs in ((common.RESAMPLE_BILINEAR, common.RESAMPLE_BICUBIC) if name in geometric else (0,)):
                    cases.append((op, m, negate, rs))
    return cases


def main():
    fill = tuple(min(255, round(255 * x)) for x in MEAN)
    seeds = []
    for seed in SEEDS:
        image = make_image(seed, 224, 224)
        out, _ = reference_sample(image, seed)
        sample, _ = uint8_sample(image, seed)
        ops, f, aff = record(sample)
        seeds.append({'seed': seed, 'ops': torch.from_numpy(ops), 'f': torch.from_numpy(f), 'affine': torch.from_numpy(aff),
                      'out': torch.from_numpy(out.copy())})
        print('seed', seed, ops[:, :3].tolist())
    h, w = OP_SIZE
    image = make_image(100, h, w)
    ops_cases = []
    for op, m, negate, rs in op_cases():
        o, f, aff = forced_layer(op, m, negate, rs, h, w)
        out = reference_op(image, op, m, negate, rs)
        ops_cases.append({'case': (op, m, negate, rs), 'ops': torch.from_numpy(o), 'f': torch.from_numpy(f),
                          'affine': torch.from_numpy(aff), 'out': torch.from_numpy(out.copy())})
    torch.save({'randaug': RANDAUG, 'fill': fill, 'seeds': seeds, 'op_size': OP_SIZE, 'op_image_seed': 100,
                'ops': ops_cases}, FIXTURE)
    print('wrote', FIXTURE, len(ops_cases), 'op cases,', os.path.getsize(FIXTURE), 'bytes')


if __name__ == '__main__':
    main()
