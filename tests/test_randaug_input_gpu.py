"""RandAugment on the uint8 input edge (csrc/capi_input.cu saicv_u8_rand_augment): the device images are bit-identical to
oracle/randaugment.py for every op forced one at a time (both resamples, 224^2 and odd sizes), for random records at
256 x 224^2 and at the smallest batch, and to the reference's Pillow outputs in tests/golden/randaug_b200.ptr; through
CudaPrefetcher fed by a multi-worker DataLoader; and malformed records are rejected before any launch."""
import importlib.util
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import mixup as omix
from oracle import randaugment as ora

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name, file):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, 'golden', file))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mk = _load('mk_randaug', 'make_randaug_golden.py')
FILL = tuple(min(255, round(255 * x)) for x in mk.MEAN)


def _record(ops, f, aff, fill=FILL):
    return types.SimpleNamespace(randaug_ops=torch.as_tensor(np.ascontiguousarray(ops), dtype=torch.int32),
                                 randaug_f=torch.as_tensor(np.ascontiguousarray(f), dtype=torch.float32),
                                 randaug_affine=torch.as_tensor(np.ascontiguousarray(aff), dtype=torch.float64),
                                 randaug_fill=fill)


def _device(images, rec):
    from simpleaicv_pytorch_training_examples_b200 import ops
    x = torch.from_numpy(np.ascontiguousarray(images)).cuda()
    ops.u8_rand_augment(x, rec)
    return x.cpu().numpy()


def _oracle(images, rec):
    return np.stack([ora.apply(images[b], rec.randaug_ops[b].numpy(), rec.randaug_f[b].numpy(),
                               rec.randaug_affine[b].numpy(), rec.randaug_fill) for b in range(len(images))])


@pytest.mark.parametrize('h,w', [(224, 224), (37, 53), (13, 17), (2, 5)])
def test_every_forced_op_matches_the_oracle(h, w):
    cases = mk.op_cases()
    recs = [mk.forced_layer(*c, h, w) for c in cases]
    rec = _record(np.stack([r[0] for r in recs]), np.stack([r[1] for r in recs]), np.stack([r[2] for r in recs]))
    images = np.stack([mk.make_image(300 + i, h, w) for i in range(len(cases))])
    got, want = _device(images, rec), _oracle(images, rec)
    for i, c in enumerate(cases):
        assert np.array_equal(got[i], want[i]), c


def test_fixture_cases_are_bit_identical():
    fx = torch.load(os.path.join(HERE, 'golden', 'randaug_b200.ptr'), weights_only=False)
    seeds = fx['seeds']
    images = np.stack([mk.make_image(c['seed'], 224, 224) for c in seeds])
    rec = _record(torch.stack([c['ops'] for c in seeds]), torch.stack([c['f'] for c in seeds]),
                  torch.stack([c['affine'] for c in seeds]), fx['fill'])
    got = _device(images, rec)
    for i, c in enumerate(seeds):
        assert np.array_equal(got[i], c['out'].numpy()), c['seed']
    h, w = fx['op_size']
    image = mk.make_image(fx['op_image_seed'], h, w)
    cases = fx['ops']
    rec = _record(torch.stack([c['ops'] for c in cases]), torch.stack([c['f'] for c in cases]),
                  torch.stack([c['affine'] for c in cases]), fx['fill'])
    got = _device(np.stack([image] * len(cases)), rec)
    for i, c in enumerate(cases):
        assert np.array_equal(got[i], c['out'].numpy()), c['case']


@pytest.mark.parametrize('b,h,w', [(256, 224, 224), (2, 224, 224), (2, 31, 45)])
def test_random_records_match_the_oracle(b, h, w):
    from simpleaicv_pytorch_training_examples_b200.classification import common
    ra = common.Uint8RandAugment(**mk.RANDAUG)
    random.seed(b + h)
    np.random.seed(b + h)
    images = np.stack([mk.make_image(1000 + i, h, w) for i in range(b)])
    samples = [ra({'image': images[i].copy(), 'label': 0}) for i in range(b)]
    rec = _record(np.stack([s['randaug_ops'] for s in samples]), np.stack([s['randaug_f'] for s in samples]),
                  np.stack([s['randaug_affine'] for s in samples]))
    got, want = _device(images, rec), _oracle(images, rec)
    for i in range(b):
        assert np.array_equal(got[i], want[i]), (i, samples[i]['randaug_ops'].tolist())
    if b == 256:
        assert set(rec.randaug_ops[:, :, 0].flatten().tolist()) == set(range(-1, 15))


def test_odd_layer_count_ends_in_the_image_buffer():
    from simpleaicv_pytorch_training_examples_b200.classification import common
    ra = common.Uint8RandAugment(**{**mk.RANDAUG, 'num_layers': 3})
    random.seed(5)
    np.random.seed(5)
    images = np.stack([mk.make_image(i, 20, 24) for i in range(8)])
    samples = [ra({'image': images[i].copy(), 'label': 0}) for i in range(8)]
    rec = _record(np.stack([s['randaug_ops'] for s in samples]), np.stack([s['randaug_f'] for s in samples]),
                  np.stack([s['randaug_affine'] for s in samples]))
    assert np.array_equal(_device(images, rec), _oracle(images, rec))


class _Synthetic(torch.utils.data.Dataset):
    """Seeded uint8 images of one size through Uint8RandAugment + Uint8RandomErasing, as a decoded dataset would deliver
    them after RandomResizedCrop and the flip."""

    def __init__(self, n, h, w, classes):
        from simpleaicv_pytorch_training_examples_b200.classification import common
        self.images = [mk.make_image(500 + i, h, w) for i in range(n)]
        self.labels = [i % classes for i in range(n)]
        self.ra = common.Uint8RandAugment(**mk.RANDAUG)
        self.erase = common.Uint8RandomErasing(prob=0.25, mode='pixel', max_count=1)

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, i):
        return self.erase(self.ra({'image': self.images[i].copy(), 'label': self.labels[i]}))


def test_prefetcher_through_a_dataloader_matches_the_oracle():
    from simpleaicv_pytorch_training_examples_b200.classification import common
    from simpleaicv_pytorch_training_examples_b200.tools.utils import CudaPrefetcher
    classes, std = 10, (0.229, 0.224, 0.225)
    loader = torch.utils.data.DataLoader(_Synthetic(8 * 6, 40, 36, classes), batch_size=8, shuffle=False, num_workers=2,
                                         pin_memory=True, collate_fn=common.Uint8MixupCutmixClassificationCollater(
                                             num_classes=classes, pin_memory=False))
    host = []

    def tee():
        for batch in loader:
            host.append(batch)
            yield batch
    busy = torch.randn(2048, 2048, device='cuda')
    got = []
    for batch in CudaPrefetcher(tee(), normalize=(mk.MEAN, std)):
        assert set(batch) == {'image', 'label'}
        for _ in range(3):                       # the next batch is copied and augmented while this work runs
            busy = torch.tanh(busy @ busy * 1e-3)
        got.append((batch['image'] * 1.).cpu())
        got.append(batch['label'].clone().cpu())
    assert len(host) == 6 and host[0]['mixup'].randaug_ops.is_pinned()
    for i, h in enumerate(host):
        rec = h['mixup']
        images = h['image'].numpy()
        augmented = torch.from_numpy(_oracle(images, rec))
        o_img, o_soft = omix.apply(augmented, h['label'], rec, mk.MEAN, std)
        assert torch.equal(got[2 * i], o_img), i
        assert torch.equal(got[2 * i + 1], o_soft), i


def test_bad_records_are_rejected_before_any_launch():
    from simpleaicv_pytorch_training_examples_b200 import _lib, ops
    x = torch.from_numpy(np.stack([mk.make_image(i, 8, 10) for i in range(2)])).cuda()

    def rec(op=(0, 0, 0, 0), f=1.0, aff=(1., 0., 0., 0., 1., 0.), fill=FILL):
        o = np.zeros((2, 2, 4), np.int32)
        o[:, :, 0] = -1
        o[1, 1] = op
        a = np.zeros((2, 2, 6))
        a[1, 1] = aff
        fl = np.ones((2, 2), np.float32)
        fl[1, 1] = f
        return _record(o, fl, a, fill)
    bad = [(rec(op=(15, 0, 0, 0)), 'op 15'), (rec(op=(-2, 0, 0, 0)), 'op -2'),
           (rec(op=(3, 1, 0, 0)), 'resample 1'), (rec(op=(11, 4, 0, 0)), 'resample 4'),
           (rec(op=(4, 0, 9, 0)), 'iparam 9'), (rec(op=(4, 0, -1, 0)), 'iparam -1'),
           (rec(op=(5, 0, 257, 0)), 'iparam 257'), (rec(op=(6, 0, 256, 0)), 'iparam 256'),
           (rec(op=(13, 2, 0, 0), aff=(1., 0., float('nan'), 0., 1., 0.)), 'not finite'),
           (rec(op=(10, 0, 0, 0), f=float('inf')), 'not finite'),
           (rec(fill=(124, 256, 104)), 'fill')]
    for r, msg in bad:
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            ops.u8_rand_augment(x, r)
        assert _lib.launch_count() == n0, msg
    n0 = _lib.launch_count()
    ops.u8_rand_augment(x, rec(op=(1, 0, 0, 0)))          # the same call with a valid record launches
    assert _lib.launch_count() > n0
