"""RandomResizedCrop / Resize + CenterCrop + flip on the uint8 input edge (csrc/capi_input.cu saicv_u8_resample): the
device images are bit-identical to oracle/resample.py at 256 x 224^2 with ragged ImageNet-like sources (flip on and off),
on edge shapes and on evaluation windows of large sources, and to the reference's Pillow outputs in
tests/golden/resample_b200.ptz; through CudaPrefetcher fed by a two-worker DataLoader for the plain recipe, the
RandAugment + Mixup recipe and test_classification on the evaluation list; and malformed geometry is rejected before any
launch."""
import importlib.util
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import mixup as omix
from oracle import randaugment as ora
from oracle import resample as ors

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _load(name, file):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, 'golden', file))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mkra = _load('mk_randaug', 'make_randaug_golden.py')


def _common():
    from simpleaicv_pytorch_training_examples_b200.classification import common
    return common


def imagenet_like_sizes(n, seed):
    """(h, w) of n sources: ImageNet-like, mostly 500 x 375 / 375 x 500 / 500 x 333, some 200..1600 wide."""
    rng = np.random.RandomState(seed)
    common = [(375, 500), (500, 375), (333, 500), (500, 333), (400, 500), (500, 500)]
    out = []
    for _ in range(n):
        if rng.rand() < 0.7:
            out.append(common[rng.randint(len(common))])
        else:
            w = int(rng.randint(200, 1601))
            out.append((max(1, int(w * rng.uniform(0.5, 1.5))), w))
    return out


def _image(seed, h, w):
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3), dtype=np.uint8)


def _device(samples):
    from simpleaicv_pytorch_training_examples_b200 import ops
    rs = _common().pack_resample(samples)
    return ops.u8_resample(rs.data.cuda(), rs.offsets, rs.geom).cpu().numpy(), rs


def _oracle(samples):
    return np.stack([ors.apply(s['image'], s['resample_geom']) for s in samples])


def _train_samples(sizes, seed, size=224):
    common = _common()
    torch.manual_seed(seed)
    rrc, flip = common.Uint8RandomResizedCrop(resize=size), common.Uint8RandomHorizontalFlip(0.5)
    return [flip(rrc({'image': _image(seed * 1000 + i, h, w), 'label': 0})) for i, (h, w) in enumerate(sizes)]


def test_train_batch_matches_the_oracle():
    samples = _train_samples(imagenet_like_sizes(256, 0), 0)
    got, rs = _device(samples)
    assert got.shape == (256, 224, 224, 3)
    flips = rs.geom[:, 8].numpy()
    assert 0 < flips.sum() < 256
    want = _oracle(samples)
    for b in range(256):
        assert np.array_equal(got[b], want[b]), (b, rs.geom[b].tolist())


@pytest.mark.parametrize('flip', [0, 1])
def test_forced_flip_matches_the_oracle(flip):
    samples = _train_samples(imagenet_like_sizes(16, 1), 1)
    for s in samples:
        s['resample_geom'][8] = flip
    got, _ = _device(samples)
    assert np.array_equal(got, _oracle(samples))


# (src h, w), (full h, w), (top, left, out h, out w): equal sizes (the pass Pillow skips), 1-pixel axes, odd sizes,
# upscale, a downscale by more than 10 and by more than 30
EDGE = [((224, 224), (224, 224), (0, 0, 224, 224)), ((224, 300), (224, 224), (0, 0, 224, 224)),
        ((300, 224), (224, 224), (0, 0, 224, 224)), ((1, 9), (5, 5), (0, 0, 5, 5)), ((9, 1), (4, 7), (0, 0, 4, 7)),
        ((1, 1), (3, 2), (0, 0, 3, 2)), ((13, 17), (5, 3), (0, 0, 5, 3)), ((37, 53), (224, 224), (0, 0, 224, 224)),
        ((3000, 2400), (224, 224), (0, 0, 224, 224)), ((1500, 7000), (40, 200), (3, 7, 31, 33)),
        ((2, 3), (70, 45), (10, 3, 31, 33))]


@pytest.mark.parametrize('src,full,window', EDGE)
def test_edge_shapes_match_the_oracle(src, full, window):
    samples = []
    for i, flip in enumerate((0, 1)):
        g = np.array([*src, *full, *window, flip], dtype=np.int32)
        samples.append({'image': _image(77 + i, *src), 'label': 0, 'resample_geom': g})
    got, _ = _device(samples)
    assert np.array_equal(got, _oracle(samples))


def test_eval_windows_of_large_sources_match_the_oracle():
    common = _common()
    resize, crop = common.Uint8Resize(256), common.Uint8CenterCrop(224)
    sizes = [(3000, 4000), (4000, 3000), (1200, 1600), (256, 256), (224, 1000), (375, 500)]
    samples = [crop(resize({'image': _image(900 + i, h, w), 'label': 0})) for i, (h, w) in enumerate(sizes)]
    got, _ = _device(samples)
    want = _oracle(samples)
    for b in range(len(sizes)):
        assert np.array_equal(got[b], want[b]), sizes[b]


def test_fixture_cases_are_bit_identical():
    fx = torch.load(os.path.join(HERE, 'golden', 'resample_b200.ptz'), weights_only=False)
    common = _common()
    for case in fx['train']:
        top, left, h, w = case['params']
        src = case['source'].numpy()
        g = np.array([h, w, case['resize'], case['resize'], 0, 0, case['resize'], case['resize'], case['flip']], np.int32)
        got, _ = _device([{'image': np.ascontiguousarray(src[top:top + h, left:left + w]), 'resample_geom': g}])
        assert np.array_equal(got[0], case['out'].numpy()), case['seed']
    for case in fx['eval']:
        s = common.Uint8CenterCrop(case['crop'])(common.Uint8Resize(case['resize'])(
            {'image': case['source'].numpy().astype(np.float32), 'label': 0}))
        got, _ = _device([s])
        assert np.array_equal(got[0], case['out'].numpy()), case['seed']


class _Sources(torch.utils.data.Dataset):
    """Seeded integer-valued float32 sources of assorted sizes, as ILSVRC2012Dataset returns them, through a transform
    list."""

    def __init__(self, sizes, transforms, classes=10):
        self.sizes, self.transforms, self.classes = sizes, transforms, classes

    def __len__(self):
        return len(self.sizes)

    def __getitem__(self, i):
        s = {'image': _image(4000 + i, *self.sizes[i]).astype(np.float32), 'label': i % self.classes}
        for t in self.transforms:
            s = t(s)
        return s


def _through_prefetcher(dataset, collate, batch_size=8):
    from simpleaicv_pytorch_training_examples_b200.tools.utils import CudaPrefetcher
    loader = torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=False, num_workers=2, pin_memory=True,
                                         collate_fn=collate)
    host = []

    def tee():
        for batch in loader:
            host.append(batch)
            yield batch
    busy = torch.randn(2048, 2048, device='cuda')
    got = []
    for batch in CudaPrefetcher(tee(), normalize=(MEAN, STD)):
        assert set(batch) == {'image', 'label'}
        for _ in range(3):                       # the next batch is copied and resized while this work runs
            busy = torch.tanh(busy @ busy * 1e-3)
        got.append(((batch['image'] * 1.).cpu(), batch['label'].clone().cpu()))
    return host, got


def _host_oracle(rs):
    return np.stack([ors.apply(rs.data[o:o + int(g[0]) * int(g[1]) * 3].numpy().reshape(int(g[0]), int(g[1]), 3), g.numpy())
                     for o, g in zip(rs.offsets.tolist(), rs.geom)])


def _normalize(u8):
    x = torch.from_numpy(u8).float().div(255.)
    return ((x - torch.tensor(MEAN)) / torch.tensor(STD)).permute(0, 3, 1, 2).contiguous()


def test_plain_recipe_through_a_dataloader_matches_the_oracle():
    common = _common()
    sizes = imagenet_like_sizes(48, 3)
    ds = _Sources(sizes, [common.Uint8RandomResizedCrop(224), common.Uint8RandomHorizontalFlip(0.5)])
    host, got = _through_prefetcher(ds, common.Uint8ClassificationCollater(pin_memory=False))
    assert len(host) == 6 and host[0]['resample'].data.is_pinned()
    for i, h in enumerate(host):
        assert torch.equal(got[i][0], _normalize(_host_oracle(h['resample']))), i
        assert torch.equal(got[i][1], h['label'])


def test_randaugment_mixup_recipe_through_a_dataloader_matches_the_oracle():
    common = _common()
    sizes = imagenet_like_sizes(48, 4)
    ds = _Sources(sizes, [common.Uint8RandomResizedCrop(224), common.Uint8RandomHorizontalFlip(0.5),
                          common.Uint8RandAugment(**mkra.RANDAUG), common.Uint8RandomErasing(prob=0.25, mode='pixel')])
    host, got = _through_prefetcher(ds, common.Uint8MixupCutmixClassificationCollater(num_classes=10, pin_memory=False))
    for i, h in enumerate(host):
        rec = h['mixup']
        resized = _host_oracle(h['resample'])
        augmented = torch.from_numpy(np.stack([ora.apply(resized[b], rec.randaug_ops[b].numpy(), rec.randaug_f[b].numpy(),
                                                         rec.randaug_affine[b].numpy(), rec.randaug_fill)
                                               for b in range(len(resized))]))
        img, soft = omix.apply(augmented, h['label'], rec, MEAN, STD)
        assert torch.equal(got[i][0], img), i
        assert torch.equal(got[i][1], soft), i


def test_test_classification_on_the_eval_list():
    from simpleaicv_pytorch_training_examples_b200.tools import scripts
    common = _common()
    sizes = [(375, 500), (500, 375), (1200, 1600), (256, 300), (333, 500), (900, 300)] * 2
    ds = _Sources(sizes, [common.Uint8Resize(256), common.Uint8CenterCrop(224)])
    loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, num_workers=2, pin_memory=True,
                                         collate_fn=common.Uint8ClassificationCollater(pin_memory=False))
    seen = []

    class Probe(torch.nn.Module):
        def forward(self, x):
            seen.append(x.clone().cpu())
            return x.float().mean(dim=(2, 3)).repeat(1, 4)

    config = types.SimpleNamespace(device_normalize=(MEAN, STD), group=None)
    acc1, acc5, loss = scripts.test_classification(loader, Probe(), torch.nn.CrossEntropyLoss(), config)
    assert len(seen) == 3 and 0 <= acc1 <= acc5 <= 100 and np.isfinite(loss)
    for i, x in enumerate(seen):
        samples = [ds[4 * i + b] for b in range(4)]
        assert torch.equal(x, _normalize(_oracle(samples))), i


def test_bad_geometry_is_rejected_before_any_launch():
    from simpleaicv_pytorch_training_examples_b200 import _lib, ops
    src = torch.from_numpy(_image(1, 10, 12)).reshape(-1).cuda()

    def call(off=0, geom=(10, 12, 8, 8, 0, 0, 8, 8, 0), n_src=None):
        g = torch.tensor([geom], dtype=torch.int32)
        s = src if n_src is None else src[:n_src]
        return ops.u8_resample(s, torch.tensor([off], dtype=torch.int64), g)
    bad = [(dict(off=3), 'past the packed buffer'), (dict(off=-1), 'past the packed buffer'),
           (dict(n_src=359), 'past the packed buffer'), (dict(geom=(0, 12, 8, 8, 0, 0, 8, 8, 0)), 'empty'),
           (dict(geom=(10, 12, 8, 0, 0, 0, 8, 8, 0)), 'empty'), (dict(geom=(10, 12, 8, 8, 1, 0, 8, 8, 0)), 'leaves'),
           (dict(geom=(10, 12, 8, 8, 0, -1, 8, 8, 0)), 'leaves'), (dict(geom=(10, 12, 8, 8, 0, 0, 8, 8, 2)), 'flip'),
           (dict(geom=(5000, 5000, 1, 1, 0, 0, 1, 1, 0), n_src=None), 'past the packed buffer')]
    for kwargs, msg in bad:
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            call(**kwargs)
        assert _lib.launch_count() == n0, msg
    huge = torch.zeros(1, 2, 2_000_000, 3, dtype=torch.uint8).reshape(-1).cuda()
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match='shared memory|taps'):
        ops.u8_resample(huge, torch.zeros(1, dtype=torch.int64), torch.tensor([[2, 2_000_000, 1, 1, 0, 0, 1, 1, 0]],
                                                                             dtype=torch.int32))
    assert _lib.launch_count() == n0
    n0 = _lib.launch_count()
    call()                                                 # the same call with valid geometry launches
    assert _lib.launch_count() > n0
