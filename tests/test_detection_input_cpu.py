"""DETR and SAM-encoder inputs on the uint8 edge, host side: oracle/detection_input.py equals cv2 run without IPP bit for
bit over up- and downscales and signed fractional translations, and stays within a measured bound of the default cv2;
the Uint8* chains consume the reference's np.random draws and give every non-image key, the recorded geometry and (via
the oracle, with cv2's IPP off) the image batch and mask of the live reference (skipped without oracle/_ref); the
committed fixture still matches the oracle; unimplemented options are refused."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import detection_input as od

cv2 = pytest.importorskip('cv2')
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_detection_input', os.path.join(HERE, 'golden', 'make_detection_input_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)

# (h, w, out_h, out_w): COCO 640 x 480 -> 1024, SA-1B-like 1500 x 2250, inexact ratios both ways, an exact 2x downscale,
# identity, tiny and 1-pixel sources
RESIZES = [(480, 640, 768, 1024), (1500, 2250, 683, 1024), (333, 500, 683, 1024), (480, 640, 683, 910), (100, 37, 1024, 379),
           (1024, 768, 1024, 768), (2048, 1536, 1024, 768), (7, 5, 3, 2), (1, 1, 5, 9), (300, 200, 41, 27), (61, 47, 128, 99)]
SHIFTS = [(10.3, -5.7), (-100.123456789, 33.015625), (0.0, 0.0), (-0.015625, 0.0078125), (500.5, -300.25), (-0.49, 0.51)]
# the largest |cv2 with IPP - oracle| measured on the 0..255 scale over RESIZES (0.0147 for 1500 x 2250 -> 683 x 1024)
IPP_BOUND = 0.02


class _ipp:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.was = cv2.ipp.useIPP()
        cv2.ipp.setUseIPP(self.on)

    def __exit__(self, *exc):
        cv2.ipp.setUseIPP(self.was)


def _u8(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)


@pytest.mark.parametrize('h,w,oh,ow', RESIZES)
def test_resize_oracle_equals_cv2_without_ipp(h, w, oh, ow):
    src = _u8(h, w, h * w).astype(np.float32)
    with _ipp(False):
        ref = cv2.resize(src, (ow, oh))
    assert np.array_equal(od.resize(src, oh, ow).view(np.int32), ref.view(np.int32))
    with _ipp(True):
        ref = cv2.resize(src, (ow, oh))
    assert np.abs(od.resize(src, oh, ow) - ref).max() <= IPP_BOUND


@pytest.mark.parametrize('tx,ty', SHIFTS)
@pytest.mark.parametrize('h,w', [(480, 640), (37, 53)])
def test_translate_oracle_equals_cv2(h, w, tx, ty):
    src = _u8(h, w, 7)
    for ipp in (False, True):
        with _ipp(ipp):
            ref = cv2.warpAffine(src.astype(np.float32), np.array([[1, 0, tx], [0, 1, ty]]), (w, h))
        assert np.array_equal(od.translate(src, tx, ty).view(np.int32), ref.view(np.int32)), ipp
    # translated, then resized: the resize of the translated float32 image
    with _ipp(False):
        ref = cv2.resize(cv2.warpAffine(src.astype(np.float32), np.array([[1, 0, tx], [0, 1, ty]]), (w, h)), (w * 3 // 2, h * 3 // 2))
    assert np.array_equal(od.resized(src, h * 3 // 2, w * 3 // 2, (tx, ty)).view(np.int32), ref.view(np.int32))


def _reference():
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    ref_import._ensure_path()
    from SimpleAICV.detection import common as rdet
    from SimpleAICV.interactive_segmentation import common as rsam
    return rdet, rsam


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


DETR_SHAPES = [(48, 64), (64, 48), (128, 100), (75, 61), (30, 100), (128, 128), (150, 90), (20, 33), (128, 40), (3, 200)]


@pytest.mark.parametrize('seed', range(24))
def test_detr_chain_matches_reference(seed):
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    rdet, _ = _reference()
    rng = np.random.RandomState(seed)
    shapes = [DETR_SHAPES[(seed + i) % len(DETR_SHAPES)] for i in range(4)]
    samples = [mk.detr_sample(rng, h, w, empty=(i == seed % 5)) for i, (h, w) in enumerate(shapes)]
    with _ipp(False):
        ref, ref_state = mk.run(samples, mk.detr_chain(rdet, 128), rdet.DETRDetectionCollater(resize=128, resize_type='yolo_style'), seed)
    ours, state = mk.run(samples, mk.detr_chain(udet, 128, 'Uint8'),
                         udet.Uint8DETRDetectionCollater(resize=128, resize_type='yolo_style', pin_memory=False), seed)
    assert _state_equal(state, ref_state), 'different np.random draws'
    for k in ('annots', 'scaled_annots'):
        assert torch.equal(ours[k], ref[k]), k
    for k in ('scale', 'size', 'scaled_size'):
        assert ours[k].dtype == ref[k].dtype and np.array_equal(ours[k], ref[k]), k
    rp = ours['resize_pad']
    assert np.array_equal(rp.geom.numpy()[:, 2:4], ref['scaled_size'].astype(np.int32))
    image, mask = mk.oracle_batch(rp)
    assert np.array_equal(mask, ref['mask'].numpy())
    assert np.array_equal(image.view(np.int32), ref['image'].contiguous().numpy().view(np.int32))


@pytest.mark.parametrize('seed', range(12))
def test_sam_chain_matches_reference(seed):
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import common as usam
    _, rsam = _reference()
    rng = np.random.RandomState(seed)
    shapes = [DETR_SHAPES[(2 * seed + i) % len(DETR_SHAPES)] for i in range(4)]
    samples = [mk.sam_sample(rng, max(h, 16), max(w, 16)) for h, w in shapes]
    with _ipp(False):
        ref, ref_state = mk.run(samples, mk.sam_chain(rsam, 128), rsam.SAMBatchCollater(resize=128), seed)
    ours, state = mk.run(samples, mk.sam_chain(usam, 128, 'Uint8'), usam.Uint8SAMBatchCollater(resize=128, pin_memory=False), seed)
    assert _state_equal(state, ref_state), 'different np.random draws'
    for k in ('box', 'mask', 'prompt_point', 'prompt_box', 'prompt_mask'):
        assert torch.equal(ours[k], ref[k]), k
    assert ours['size'].dtype == ref['size'].dtype and np.array_equal(ours['size'], ref['size'])
    rp = ours['resize_pad']
    image, _ = mk.oracle_batch(rp)
    assert np.array_equal(image.view(np.int32), ref['image'].contiguous().numpy().view(np.int32))


def test_detr_chain_covers_every_branch():
    """Over the seeds of test_detr_chain_matches_reference: flip, crop and translate fire and do not, and both
    multi-scale sizes are drawn."""
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    translated, sizes = set(), set()
    for seed in range(24):
        rng = np.random.RandomState(seed)
        shapes = [DETR_SHAPES[(seed + i) % len(DETR_SHAPES)] for i in range(4)]
        samples = [mk.detr_sample(rng, h, w, empty=(i == seed % 5)) for i, (h, w) in enumerate(shapes)]
        ours, _ = mk.run(samples, mk.detr_chain(udet, 128, 'Uint8'),
                         udet.Uint8DETRDetectionCollater(resize=128, resize_type='yolo_style', pin_memory=False), seed)
        g = ours['resize_pad'].geom.numpy()
        translated |= set(g[:, 5].tolist())
        sizes |= set(int(v) for v in g[:, 2:4].max(1))
    assert translated == {0, 1} and sizes == {96, 128}


def test_fixture_matches_oracle():
    z = np.load(mk.FIXTURE)
    from simpleaicv_pytorch_training_examples_b200.detection.common import ResizePadBatch
    for kind, batches in (('detr', mk.DETR_BATCHES), ('sam', mk.SAM_BATCHES)):
        for seed, _ in batches:
            p = f'{kind}{seed}_'
            norm = (None, None) if kind == 'detr' else ((123.675, 116.28, 103.53), (58.395, 57.12, 57.375))
            rp = ResizePadBatch(torch.from_numpy(z[p + 'data']), torch.from_numpy(z[p + 'offsets']), torch.from_numpy(z[p + 'geom']),
                                torch.from_numpy(z[p + 'shift']), mk.RESIZE, *norm)
            image, mask = mk.oracle_batch(rp)
            assert np.array_equal(image.view(np.int32), z[p + 'oracle_image'].view(np.int32)), p
            assert np.array_equal(mask, z[p + 'oracle_mask']), p
            # the reference as shipped (cv2 with IPP) differs from the oracle by resize rounding only, normalised here
            assert np.abs(z[p + 'ref_image'] - image).max() <= (IPP_BOUND / 255 if kind == 'detr' else IPP_BOUND / 57), p
            if kind == 'detr':
                assert np.array_equal(z[p + 'ref_mask'], mask), p


def test_unimplemented_options_are_refused():
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    with pytest.raises(NotImplementedError):
        udet.Uint8DetectionResize(resize=1024, resize_type='retina_style')
    s = mk.detr_sample(np.random.RandomState(0), 40, 50, empty=False)
    s = udet.Uint8DetectionResize(resize=64, resize_type='yolo_style')(s)
    with pytest.raises(ValueError):
        udet.Uint8RandomCrop(prob=1.0)(s)
    with pytest.raises(ValueError):       # no Uint8Normalize
        udet.Uint8DETRDetectionCollater(resize=64, pin_memory=False)([s])
