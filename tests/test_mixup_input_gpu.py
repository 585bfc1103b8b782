"""Mixup / CutMix + RandomErasing on the uint8 input edge (csrc/capi_input.cu saicv_u8_mix_erase_norm): device images and
soft labels are bit-identical to oracle/mixup.py and to the reference's batches in tests/golden/mixup_erase_b6.ptu, at
224^2 x 256, at the smallest batch and on the scalar path; through CudaPrefetcher fed by a multi-worker DataLoader; and
malformed draws are rejected before any launch."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import mixup as omix

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_mixup', os.path.join(HERE, 'golden', 'make_mixup_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


def _device(batch, **kw):
    from simpleaicv_pytorch_training_examples_b200 import ops
    rec = batch['mixup']
    return ops.u8_mix_erase_normalize(batch['image'].cuda(), batch['label'].cuda(), mk.MEAN, mk.STD, rec, rec.noise.cuda(), **kw)


def test_fixture_cases_are_bit_identical():
    fx = torch.load(os.path.join(HERE, 'golden', 'mixup_erase_b6.ptu'), weights_only=False)
    for case in fx['cases']:
        batch, _ = mk.uint8_batch(case['images'].numpy(), case['labels'].tolist(), case['seed'], **case['collate'])
        img, soft = _device(batch)
        torch.cuda.synchronize()
        assert torch.equal(img.cpu(), case['image']), case['name']
        assert torch.equal(soft.cpu(), case['label']), case['name']
        o_img, o_soft = omix.apply(batch['image'], batch['label'], batch['mixup'], mk.MEAN, mk.STD)
        assert torch.equal(img.cpu(), o_img) and torch.equal(soft.cpu(), o_soft), case['name']


@pytest.mark.parametrize('b,h,w,classes', [(256, 224, 224, 1000), (2, 32, 48, 10), (4, 9, 13, 10), (6, 15, 7, 7)])
def test_kernel_matches_oracle(b, h, w, classes):
    from simpleaicv_pytorch_training_examples_b200.classification import common
    images, labels = mk.make_inputs(b * 100 + h, b, h, w, classes)
    seen = set()
    for seed in range(200):
        batch, _ = mk.uint8_batch(images, labels, seed, num_classes=classes)
        rec = batch['mixup']
        if rec.mode in seen or (b > 2 and not (rec.rects[:, 2] > 0).any()):
            continue
        seen.add(rec.mode)
        img, soft = _device(batch)
        o_img, o_soft = omix.apply(batch['image'], batch['label'], rec, mk.MEAN, mk.STD)
        assert img.shape == (b, 3, h, w) and soft.shape == (b, classes)
        assert torch.equal(img.cpu(), o_img), (seed, rec.mode)
        assert torch.equal(soft.cpu(), o_soft), (seed, rec.mode)
        if seen == {common.MIX_MIXUP, common.MIX_CUTMIX}:
            break
    assert seen == {common.MIX_MIXUP, common.MIX_CUTMIX}


class _Synthetic(torch.utils.data.Dataset):
    """Seeded uint8 images of one size through Uint8RandomErasing, as a decoded dataset would deliver them."""

    def __init__(self, n, h, w, classes):
        from simpleaicv_pytorch_training_examples_b200.classification import common
        self.images, self.labels = mk.make_inputs(77, n, h, w, classes)
        self.erase = common.Uint8RandomErasing(prob=0.5, mode='pixel', max_count=1)

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, i):
        return self.erase({'image': self.images[i].copy(), 'label': self.labels[i]})


def test_prefetcher_through_a_dataloader_matches_the_oracle():
    from simpleaicv_pytorch_training_examples_b200.classification import common
    from simpleaicv_pytorch_training_examples_b200.tools.utils import CudaPrefetcher
    classes = 10
    loader = torch.utils.data.DataLoader(_Synthetic(8 * 7, 40, 36, classes), batch_size=8, shuffle=False, num_workers=2,
                                         pin_memory=True, collate_fn=common.Uint8MixupCutmixClassificationCollater(
                                             num_classes=classes, pin_memory=False))
    host = []

    def tee():
        for batch in loader:
            host.append(batch)
            yield batch
    busy = torch.randn(2048, 2048, device='cuda')
    got = []
    for i, batch in enumerate(CudaPrefetcher(tee(), normalize=(mk.MEAN, mk.STD))):
        assert set(batch) == {'image', 'label'}
        assert batch['image'].dtype == torch.float32 and batch['label'].shape == (8, classes)
        for _ in range(3):                       # the next batch is copied and mixed while this work runs
            busy = torch.tanh(busy @ busy * 1e-3)
        got.append((batch['image'] * 1.).cpu())
        got.append(batch['label'].clone().cpu())
    assert len(host) == 7 and len(got) == 14
    assert host[0]['image'].is_pinned() and host[0]['mixup'].noise.is_pinned()
    assert len({int(h['mixup'].noise.numel()) for h in host}) > 1          # the noise length changed between batches
    for i, h in enumerate(host):
        o_img, o_soft = omix.apply(h['image'], h['label'], h['mixup'], mk.MEAN, mk.STD)
        assert torch.equal(got[2 * i], o_img), i
        assert torch.equal(got[2 * i + 1], o_soft), i


def test_prefetcher_without_normalize_raises():
    from simpleaicv_pytorch_training_examples_b200.tools.utils import CudaPrefetcher
    images, labels = mk.make_inputs(0, 4, 8, 8)
    batch, _ = mk.uint8_batch(images, labels, 0)
    with pytest.raises(RuntimeError, match='normalize'):
        next(iter(CudaPrefetcher([batch])))


def test_bad_draws_are_rejected_before_any_launch():
    from simpleaicv_pytorch_training_examples_b200 import _lib
    from simpleaicv_pytorch_training_examples_b200.classification import common
    images, labels = mk.make_inputs(1, 4, 8, 10)
    x, y = torch.from_numpy(images).cuda(), torch.tensor(labels).cuda()
    noise = torch.zeros(64, device='cuda')
    from simpleaicv_pytorch_training_examples_b200 import ops

    def rec(rects=((0, 0, 0, 0),) * 4, offsets=(0, 0, 0, 0), used=64, mode=common.MIX_MIXUP, box=(0, 0, 0, 0), lam=0.5):
        return common.MixupEraseRecord(torch.tensor(rects, dtype=torch.int32), torch.tensor(offsets, dtype=torch.int64),
                                       torch.zeros(used), mode, box, lam, 10, 0.91, 0.01)
    bad = [(rec(rects=((0, 0, 0, 0), (5, 0, 4, 2), (0, 0, 0, 0), (0, 0, 0, 0))), 'leaves'),        # rows 5..8 of 8
           (rec(rects=((0, 0, 0, 0), (0, 9, 2, 2), (0, 0, 0, 0), (0, 0, 0, 0))), 'leaves'),        # columns 9..10 of 10
           (rec(rects=((0, 0, 0, 0), (-1, 0, 2, 2), (0, 0, 0, 0), (0, 0, 0, 0))), 'negative'),
           (rec(rects=((0, 0, 0, 0), (0, 0, 4, 4), (0, 0, 0, 0), (0, 0, 0, 0)), offsets=(0, 20, 0, 0)), 'past the buffer'),
           (rec(rects=((0, 0, 0, 0), (0, 0, 2, 2), (0, 0, 0, 0), (0, 0, 0, 0)), offsets=(0, -4, 0, 0)), 'past the buffer'),
           (rec(lam=float('nan')), 'not finite'),
           (rec(lam=float('inf')), 'not finite'),
           (rec(mode=common.MIX_CUTMIX, box=(0, 9, 0, 4)), 'box'),
           (rec(mode=common.MIX_CUTMIX, box=(3, 2, 0, 4)), 'box'),
           (rec(mode=7), 'mode')]
    for r, msg in bad:
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            ops.u8_mix_erase_normalize(x, y, mk.MEAN, mk.STD, r, noise)
        assert _lib.launch_count() == n0, msg
    n0 = _lib.launch_count()
    odd = common.MixupEraseRecord(torch.zeros(3, 4, dtype=torch.int32), torch.zeros(3, dtype=torch.int64), torch.zeros(0),
                                  common.MIX_MIXUP, (0, 0, 0, 0), 0.5, 10, 0.91, 0.01)
    with pytest.raises(RuntimeError, match='even'):
        ops.u8_mix_erase_normalize(x[:3].contiguous(), y[:3].contiguous(), mk.MEAN, mk.STD, odd, noise)
    assert _lib.launch_count() == n0
    ops.u8_mix_erase_normalize(x, y, mk.MEAN, mk.STD, rec(), noise)      # the same call with valid draws launches
    assert _lib.launch_count() == n0 + 2
