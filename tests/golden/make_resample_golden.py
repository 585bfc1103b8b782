"""Generates tests/golden/resample_b200.ptz by running the REFERENCE geometric transforms of the ImageNet recipes, through
torchvision and Pillow, on seeded synthetic images of assorted shapes:

- train: Opencv2PIL -> TorchRandomResizedCrop(resize) -> TorchRandomHorizontalFlip(0.5)
  (SimpleAICV/classification/common.py:22-37,58-75,97-112), each case from torch.manual_seed(seed);
- eval: Opencv2PIL -> TorchResize(resize) -> TorchCenterCrop(crop) (:154-187).

The transforms receive integer-valued float32 sources, as ILSVRC2012Dataset returns them; the fixture stores them as
uint8 (the same values).  Per case it holds the source, the seed, the
drawn crop (top, left, h, w) and flip, the reference's uint8 output and torch's generator state after the transforms.
It pins oracle/resample.py and the device kernel without the reference.  The file is not a .pt: tests/test_oracle_golden.py
loads every *.pt as a network fixture.

    python tests/golden/make_resample_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

FIXTURE = os.path.join(HERE, 'resample_b200.ptz')
# (seed, (h, w), resize): downscale, upscale, a tiny source that reaches the 10-try fallback, extreme aspect ratios.
# The sizes are small so that the file stays small; the GPU tests run the shipped 224 against the oracle this pins.
TRAIN = [(0, (75, 100), 64), (1, (61, 47), 48), (2, (60, 80), 40), (3, (7, 5), 32), (4, (12, 180), 32),
         (5, (180, 11), 32), (6, (49, 66), 40), (7, (64, 48), 56)]
# (seed, (h, w), resize, crop): short side larger or smaller than the resize, portrait and landscape
EVAL = [(10, (90, 68), 56, 48), (11, (30, 53), 40, 36), (12, (40, 40), 40, 32), (13, (19, 134), 24, 20)]


def make_source(seed, h, w):
    """Integer-valued float32 [h, w, 3], the dtype the dataset's decode path returns."""
    rng = np.random.RandomState(30_000 + seed)
    coarse = rng.uniform(0, 255, size=((h + 5) // 6 + 1, (w + 5) // 6 + 1, 3))
    field = np.repeat(np.repeat(coarse, 6, 0), 6, 1)[:h, :w]
    return np.clip(np.round(field + rng.normal(0, 20, size=(h, w, 3))), 0, 255).astype(np.float32)


def reference_train(image, seed, resize):
    """(uint8 output, (top, left, h, w), flip, torch state) of the reference's train transforms from torch seed."""
    import torchvision.transforms as T
    from baseline import ref_import
    ref = ref_import.module('SimpleAICV.classification.common')
    drawn = []
    get_params = T.RandomResizedCrop.get_params

    def logged(*args, **kwargs):
        drawn.append(get_params(*args, **kwargs))
        return drawn[-1]
    torch.manual_seed(seed)
    T.RandomResizedCrop.get_params = staticmethod(logged)
    try:
        s = {'image': image.copy(), 'label': 0}
        for t in (ref.Opencv2PIL(), ref.TorchRandomResizedCrop(resize=resize)):
            s = t(s)
        cropped = np.asarray(s['image'])
        s = ref.TorchRandomHorizontalFlip(prob=0.5)(s)
    finally:
        T.RandomResizedCrop.get_params = staticmethod(get_params)
    out = np.asarray(s['image'])
    return out, drawn[0], int(not np.array_equal(out, cropped)), torch.get_rng_state()


def reference_eval(image, resize, crop):
    from baseline import ref_import
    ref = ref_import.module('SimpleAICV.classification.common')
    s = {'image': image.copy(), 'label': 0}
    for t in (ref.Opencv2PIL(), ref.TorchResize(resize=resize), ref.TorchCenterCrop(resize=crop)):
        s = t(s)
    return np.asarray(s['image'])


def main():
    train, evals = [], []
    for seed, (h, w), resize in TRAIN:
        image = make_source(seed, h, w)
        out, params, flip, state = reference_train(image, seed, resize)
        train.append({'seed': seed, 'resize': resize, 'source': torch.from_numpy(image.astype(np.uint8)), 'params': params, 'flip': flip,
                      'out': torch.from_numpy(out.copy()), 'torch_state': state})
        print('train', seed, (h, w), params, flip)
    for seed, (h, w), resize, crop in EVAL:
        image = make_source(seed, h, w)
        evals.append({'seed': seed, 'resize': resize, 'crop': crop,
                      'source': torch.from_numpy(image.astype(np.uint8)),
                      'out': torch.from_numpy(reference_eval(image, resize, crop).copy())})
        print('eval', seed, (h, w), resize, crop)
    torch.save({'train': train, 'eval': evals}, FIXTURE)
    print('wrote', FIXTURE, os.path.getsize(FIXTURE), 'bytes')


if __name__ == '__main__':
    main()
