"""Mixup / CutMix + RandomErasing on the uint8 input edge, host side: Uint8RandomErasing + Uint8MixupCutmixClassification-
Collater make the reference's np.random draws in its order (checked against the live reference, skipped without
oracle/_ref), oracle/mixup.py applied to their record reproduces the reference's batch bit for bit (live, and against the
committed reference fixture), and inputs or options the edge does not implement are rejected."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import mixup as omix
from simpleaicv_pytorch_training_examples_b200.classification import common

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_mixup', os.path.join(HERE, 'golden', 'make_mixup_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


def _fixture():
    return torch.load(os.path.join(HERE, 'golden', 'mixup_erase_b6.ptu'), weights_only=False)


def test_fixture_pins_the_draws_and_the_oracle():
    fx = _fixture()
    assert [c['name'] for c in fx['cases']] == [name for name, _, _ in mk.CASES]
    for case in fx['cases']:
        images, labels = case['images'].numpy(), case['labels'].tolist()
        with mk.draw_log() as log:
            batch, _ = mk.uint8_batch(images, labels, case['seed'], **case['collate'])
        rec = batch['mixup']
        h, w = images.shape[1:3]
        assert mk._case_holds(case['name'], rec, log, h, w), case['name']
        assert batch['image'].dtype == torch.uint8 and torch.equal(batch['image'], case['images'])
        assert torch.equal(batch['label'], case['labels'])
        img, soft = omix.apply(batch['image'], batch['label'], rec, fx['mean'], fx['std'])
        assert torch.equal(img, case['image']), case['name']
        assert torch.equal(soft, case['label']), case['name']


# (batch, h, w, collater overrides): the shipped arguments at even / odd pixel counts, plus the other branches of the draws
CONFIGS = [(6, 10, 14, {}), (8, 9, 13, {}), (4, 16, 12, {}), (2, 7, 5, {}),
           (6, 10, 14, {'mixup_cutmix_prob': 0.5}), (6, 12, 10, {'cutmix_alpha': 0.}), (6, 12, 10, {'mixup_alpha': 0.}),
           (6, 11, 15, {'correct_lam': False, 'label_smoothing': 0.})]


@pytest.mark.parametrize('b,h,w,collate', CONFIGS)
def test_draws_state_and_batch_match_the_live_reference(b, h, w, collate):
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    seeds = range(50) if not collate else range(12)
    modes = set()
    for seed in seeds:
        images, labels = mk.make_inputs(seed, b, h, w)
        with mk.draw_log() as ref_log:
            ref, ref_state = mk.reference_batch(images, labels, seed, **collate)
        with mk.draw_log() as log:
            got, state = mk.uint8_batch(images, labels, seed, **collate)
        assert [n for n, _ in log] == [n for n, _ in ref_log], seed
        assert all(np.array_equal(a, r) for (_, a), (_, r) in zip(log, ref_log)), seed
        assert state[0] == ref_state[0] and np.array_equal(state[1], ref_state[1]) and state[2:] == ref_state[2:], seed
        rec = got['mixup']
        modes.add(rec.mode)
        img, soft = omix.apply(got['image'], got['label'], rec, mk.MEAN, mk.STD)
        assert torch.equal(img, ref['image'].contiguous()), seed
        assert soft.dtype == ref['label'].dtype == torch.float32 and torch.equal(soft, ref['label']), seed
    if not collate:
        assert modes == {common.MIX_MIXUP, common.MIX_CUTMIX}


def _samples(b=4, h=8, w=10, labels=None):
    images, lab = mk.make_inputs(0, b, h, w)
    erase = common.Uint8RandomErasing(**mk.ERASE)
    return [erase({'image': images[i], 'label': (labels or lab)[i]}) for i in range(b)]


def test_record_layout():
    np.random.seed(3)
    samples = _samples(b=8, h=16, w=12)
    batch = common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False)(samples)
    rec = batch['mixup']
    assert set(batch) == {'image', 'label', 'mixup'}
    assert batch['image'].shape == (8, 16, 12, 3) and batch['image'].dtype == torch.uint8
    assert batch['label'].dtype == torch.int64
    assert rec.rects.dtype == torch.int32 and rec.rects.shape == (8, 4)
    assert rec.offsets.dtype == torch.int64 and rec.noise.dtype == torch.float32
    sizes = (rec.rects[:, 2] * rec.rects[:, 3] * 3).tolist()
    assert rec.offsets.tolist() == [sum(sizes[:i]) for i in range(8)] and rec.noise.numel() == sum(sizes)
    for s, r in zip(samples, rec.rects):
        assert s['image'].dtype == np.uint8 and tuple(s['erase_rect']) == tuple(r.tolist())


def test_rejects_bad_batches():
    collate = common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False)
    with pytest.raises(ValueError, match='even'):
        collate(_samples(b=3))
    with pytest.raises(ValueError, match='labels'):
        collate(_samples(labels=[0, 1, 10, 2]))
    with pytest.raises(ValueError, match='labels'):
        collate(_samples(labels=[0, -1, 3, 2]))
    mixed = _samples()
    mixed[1] = _samples(h=8, w=9)[1]
    with pytest.raises(ValueError, match='one shape'):
        collate(mixed)
    with pytest.raises(ValueError):
        common.Uint8RandomErasing()({'image': np.zeros((4, 4, 3), np.float32), 'label': 0})


@pytest.mark.parametrize('kwargs', [{'mode': 'pair'}, {'mode': 'elem'}, {'cutmix_minmax': (0.2, 0.8)}, {'use_mixup': False}])
def test_unimplemented_collater_options_raise(kwargs):
    with pytest.raises(NotImplementedError, match='shipped'):
        common.Uint8MixupCutmixClassificationCollater(**kwargs)


@pytest.mark.parametrize('kwargs', [{'mode': 'const'}, {'mode': 'rand'}, {'max_count': 2}, {'min_count': 2, 'max_count': 2}])
def test_unimplemented_erase_options_raise(kwargs):
    with pytest.raises(NotImplementedError, match='shipped'):
        common.Uint8RandomErasing(**kwargs)
