"""RandAugment on the uint8 input edge, host side: Uint8RandAugment makes the reference RandAugment's random / np.random
draws in its order (checked against the live reference, skipped without oracle/_ref), oracle/randaugment.py applied to
its record reproduces the reference's Pillow output bit for bit (live, per op and for whole calls, and against the
committed reference fixture), the whole ImageNet train chain gives the reference's fp32 batch, and options or samples
the edge does not implement are rejected."""
import importlib.util
import os
import random

import numpy as np
import pytest
import torch

from oracle import mixup as omix
from oracle import randaugment as ora
from simpleaicv_pytorch_training_examples_b200.classification import common

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name, file):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, 'golden', file))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mk = _load('mk_randaug', 'make_randaug_golden.py')
mkmix = _load('mk_mixup', 'make_mixup_golden.py')
FILL = (124, 116, 104)


def _reference():
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    return ref_import


def _apply(sample):
    return ora.apply(sample['image'], sample['randaug_ops'], sample['randaug_f'], sample['randaug_affine'],
                     sample['randaug_fill'])


def test_fixture_pins_the_draws_and_the_oracle():
    fx = torch.load(os.path.join(HERE, 'golden', 'randaug_b200.ptr'), weights_only=False)
    assert fx['fill'] == FILL and [c['seed'] for c in fx['seeds']] == list(mk.SEEDS)
    for case in fx['seeds']:
        sample, _ = mk.uint8_sample(mk.make_image(case['seed'], 224, 224), case['seed'])
        assert np.array_equal(sample['randaug_ops'], case['ops'].numpy()), case['seed']
        assert np.array_equal(sample['randaug_f'], case['f'].numpy()), case['seed']
        assert np.array_equal(sample['randaug_affine'], case['affine'].numpy()), case['seed']
        assert np.array_equal(_apply(sample), case['out'].numpy()), case['seed']
    h, w = fx['op_size']
    image = mk.make_image(fx['op_image_seed'], h, w)
    assert [c['case'] for c in fx['ops']] == mk.op_cases()
    for case in fx['ops']:
        ops, f, aff = mk.forced_layer(*case['case'], h, w)
        assert np.array_equal(ops, case['ops'].numpy()) and np.array_equal(f, case['f'].numpy()), case['case']
        assert np.array_equal(aff, case['affine'].numpy()), case['case']
        assert np.array_equal(ora.apply(image, ops, f, aff, FILL), case['out'].numpy()), case['case']


def test_draws_state_and_output_match_the_live_reference():
    _reference()
    ops_seen = set()
    for seed in range(240):
        h, w = (224, 224) if seed % 4 == 0 else (37, 53)
        image = mk.make_image(seed, h, w)
        ref, ref_state = mk.reference_sample(image, seed)
        sample, state = mk.uint8_sample(image, seed)
        assert state[0] == ref_state[0], seed
        assert all(np.array_equal(a, b) for a, b in zip(state[1], ref_state[1])), seed
        assert sample['image'].dtype == np.uint8 and np.array_equal(sample['image'], image)
        assert np.array_equal(_apply(sample), ref), (seed, sample['randaug_ops'].tolist())
        ops_seen.update(int(o) for o in sample['randaug_ops'][:, 0])
    assert ops_seen == set(range(-1, 15))


def test_draws_without_magnitude_noise_match_the_live_reference():
    ref_import = _reference()
    ar = ref_import.module('SimpleAICV.classification.auto_rand_augment')
    from PIL import Image
    for seed in range(40):
        image = mk.make_image(seed, 19, 23)
        random.seed(seed)
        np.random.seed(seed)
        ref = np.asarray(ar.RandAugment(**{**mk.RANDAUG, 'magnitude_std': 0, 'num_layers': 3, 'magnitude': 7})(
            {'image': Image.fromarray(image), 'label': 0})['image'])
        ref_state = random.getstate(), np.random.get_state()
        sample, state = mk.uint8_sample(image, seed, magnitude_std=0, num_layers=3, magnitude=7)
        assert state[0] == ref_state[0] and all(np.array_equal(a, b) for a, b in zip(state[1], ref_state[1])), seed
        assert np.array_equal(_apply(sample), ref), seed


@pytest.mark.parametrize('h,w', [(224, 224), (37, 53)])
def test_oracle_matches_pillow_for_every_forced_op(h, w):
    _reference()
    image = mk.make_image(7, h, w)
    for case in mk.op_cases():
        ops, f, aff = mk.forced_layer(*case, h, w)
        assert np.array_equal(ora.apply(image, ops, f, aff, FILL), mk.reference_op(image, *case)), case


def _chain(seed, images, labels, ours):
    """One batch of the ImageNet train chain from torch / random / np.random seeded with ``seed``: the reference's
    (RRC, flip, RandAugment, normalise, RandomErasing, MixupCutmixClassificationCollater) or ours (RRC, flip,
    Uint8RandAugment, Uint8RandomErasing, Uint8MixupCutmixClassificationCollater), and the three generators' states."""
    from baseline import ref_import
    ref = ref_import.module('SimpleAICV.classification.common')
    ar = ref_import.module('SimpleAICV.classification.auto_rand_augment')
    torch.manual_seed(seed)
    random.seed(seed)
    np.random.seed(seed)
    head = [ref.Opencv2PIL(), ref.TorchRandomResizedCrop(resize=40), ref.TorchRandomHorizontalFlip(prob=0.5)]
    if ours:
        tail = [common.Uint8RandAugment(**mk.RANDAUG), common.Uint8RandomErasing(**mkmix.ERASE)]
        collate = common.Uint8MixupCutmixClassificationCollater(**mkmix.COLLATE, pin_memory=False)
    else:
        tail = [ar.RandAugment(**mk.RANDAUG), ref.TorchMeanStdNormalize(mean=list(mkmix.MEAN), std=list(mkmix.STD)),
                ref.RandomErasing(**mkmix.ERASE)]
        collate = ref.MixupCutmixClassificationCollater(**mkmix.COLLATE)
    samples = []
    for i in range(len(labels)):
        s = {'image': images[i].copy(), 'label': labels[i]}
        for t in head + tail:
            s = t(s)
        samples.append(s)
    return collate(samples), (torch.get_rng_state(), random.getstate(), np.random.get_state())


def test_whole_chain_matches_the_live_reference():
    _reference()
    for seed in range(24):
        images, labels = mkmix.make_inputs(seed, 4, 57, 71)
        ref, ref_state = _chain(seed, images, labels, ours=False)
        got, state = _chain(seed, images, labels, ours=True)
        assert torch.equal(state[0], ref_state[0]) and state[1] == ref_state[1], seed
        assert all(np.array_equal(a, b) for a, b in zip(state[2], ref_state[2])), seed
        rec = got['mixup']
        assert rec.randaug_ops.shape == (4, 2, 4) and rec.randaug_fill == FILL
        augmented = torch.from_numpy(np.stack([ora.apply(got['image'][b].numpy(), rec.randaug_ops[b].numpy(),
                                                         rec.randaug_f[b].numpy(), rec.randaug_affine[b].numpy(),
                                                         rec.randaug_fill) for b in range(4)]))
        img, soft = omix.apply(augmented, got['label'], rec, mkmix.MEAN, mkmix.STD)
        assert torch.equal(img, ref['image'].contiguous()), seed
        assert torch.equal(soft, ref['label']), seed


def _samples(b=4, h=12, w=10, randaug=True):
    random.seed(0)
    np.random.seed(0)
    images, labels = mkmix.make_inputs(0, b, h, w)
    ra, erase = common.Uint8RandAugment(**mk.RANDAUG), common.Uint8RandomErasing(**mkmix.ERASE)
    return [erase(ra({'image': images[i], 'label': labels[i]}) if randaug else {'image': images[i], 'label': labels[i]})
            for i in range(b)]


def test_record_layout():
    samples = _samples(b=6)
    for s in samples:
        assert s['randaug_ops'].dtype == np.int32 and s['randaug_ops'].shape == (2, 4)
        assert s['randaug_f'].dtype == np.float32 and s['randaug_f'].shape == (2,)
        assert s['randaug_affine'].dtype == np.float64 and s['randaug_affine'].shape == (2, 6)
    rec = common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False)(samples)['mixup']
    assert rec.randaug_ops.dtype == torch.int32 and rec.randaug_ops.shape == (6, 2, 4)
    assert rec.randaug_f.dtype == torch.float32 and rec.randaug_f.shape == (6, 2)
    assert rec.randaug_affine.dtype == torch.float64 and rec.randaug_affine.shape == (6, 2, 6)
    assert rec.randaug_fill == FILL
    for b, s in enumerate(samples):
        assert np.array_equal(rec.randaug_ops[b].numpy(), s['randaug_ops'])
    plain = common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False)(_samples(randaug=False))['mixup']
    assert plain.randaug_ops is None and plain.randaug_f is None and plain.randaug_affine is None


def test_collaters_do_not_drop_or_mix_records():
    with pytest.raises(ValueError, match='RandAugment'):
        common.Uint8ClassificationCollater(pin_memory=False)(_samples())
    mixed = _samples()[:2] + _samples(randaug=False)[2:]
    with pytest.raises(ValueError, match='some samples'):
        common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False)(mixed)
    with pytest.raises(ValueError):
        common.Uint8RandAugment()({'image': np.zeros((4, 4, 3), np.float32), 'label': 0})


@pytest.mark.parametrize('kwargs', [{'integer': False}, {'weight_idx': 0}, {'magnitude_std': float('inf')},
                                    {'magnitude_max': 15}])
def test_unimplemented_options_raise(kwargs):
    with pytest.raises(NotImplementedError, match='shipped'):
        common.Uint8RandAugment(**kwargs)
