"""RandomResizedCrop / Resize + CenterCrop + flip on the uint8 input edge, host side: the Uint8* transforms make
torchvision's draws in its order from torch's global generator (checked against torchvision, and the reference chains
against the live reference, skipped without oracle/_ref), oracle/resample.py equals Pillow's bilinear resize bit for bit
(live, and against the committed reference fixture), the whole chains give the reference's fp32 batches, the collaters
pack ragged crops, unimplemented options are refused, and the resample kernel's SASS fuses no float64 multiply-add
outside the correctly rounded divisions."""
import importlib.util
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import mixup as omix
from oracle import randaugment as ora
from oracle import resample as ors
from simpleaicv_pytorch_training_examples_b200.classification import common

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _load(name, file):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, 'golden', file))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mk = _load('mk_resample', 'make_resample_golden.py')
mkra = _load('mk_randaug', 'make_randaug_golden.py')
mkmix = _load('mk_mixup', 'make_mixup_golden.py')

# source shapes of the draw tests: ImageNet-like, tiny, 1-pixel and extreme aspect ratios (the 10-try fallback)
SHAPES = [(375, 500), (500, 375), (224, 224), (7, 5), (1, 1), (1, 40), (40, 1), (20, 300), (300, 18), (61, 47), (3, 1000)]


def _reference():
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    return ref_import


def test_draws_and_generator_state_match_torchvision():
    T = pytest.importorskip('torchvision.transforms')
    Image = pytest.importorskip('PIL.Image')
    fallback = 0
    for seed in range(220):
        h, w = SHAPES[seed % len(SHAPES)]
        scale = (0.08, 1.0) if seed % 3 else (0.35, 1.0)
        img = Image.new('RGB', (w, h))
        torch.manual_seed(seed)
        want = T.RandomResizedCrop.get_params(img, list(scale), [3. / 4., 4. / 3.])
        want_flip = bool(torch.rand(1) < 0.5)
        want_state = torch.get_rng_state()
        torch.manual_seed(seed)
        s = common.Uint8RandomResizedCrop(resize=224, scale=scale)({'image': np.zeros((h, w, 3), np.float32), 'label': 0})
        s = common.Uint8RandomHorizontalFlip(0.5)(s)
        assert torch.equal(torch.get_rng_state(), want_state), seed
        top, left, ch, cw = want
        assert s['resample_geom'].tolist() == [ch, cw, 224, 224, 0, 0, 224, 224, int(want_flip)], seed
        assert s['image'].dtype == np.uint8 and s['image'].shape == (ch, cw, 3)
        fallback += _falls_back(seed, h, w, scale)
    assert fallback > 0


def _falls_back(seed, h, w, scale):
    """Whether all 10 of get_params' tries fail for this seed, so that it takes the centre-crop fallback."""
    torch.manual_seed(seed)
    log_ratio = torch.log(torch.tensor((3. / 4., 4. / 3.)))
    for _ in range(10):
        target = h * w * torch.empty(1).uniform_(*scale).item()
        ar = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        cw, ch = int(round((target * ar) ** 0.5)), int(round((target / ar) ** 0.5))
        if 0 < cw <= w and 0 < ch <= h:
            return False
    return True


def test_crop_keeps_the_pixels_and_accepts_uint8():
    image = np.random.RandomState(0).randint(0, 256, size=(50, 60, 3)).astype(np.float32)
    for src in (image, image.astype(np.uint8)):
        torch.manual_seed(3)
        s = common.Uint8RandomResizedCrop(32)({'image': src, 'label': 0})
        torch.manual_seed(3)
        top, left, h, w = common.random_resized_crop_params(50, 60, (0.08, 1.0), (3. / 4., 4. / 3.))
        assert s['image'].dtype == np.uint8 and s['image'].flags['C_CONTIGUOUS']
        assert np.array_equal(s['image'], image[top:top + h, left:left + w].astype(np.uint8))


# (src h, w), (out h, w): downscale, upscale, equal width / height / both, 1-pixel axes, odd sizes, downscale > 10
RESIZE_CASES = [((375, 500), (224, 224)), ((37, 53), (224, 224)), ((224, 300), (224, 224)), ((300, 224), (224, 224)),
                ((224, 224), (224, 224)), ((1, 9), (4, 4)), ((9, 1), (2, 7)), ((1, 1), (3, 3)), ((13, 17), (5, 3)),
                ((3000, 2600), (224, 224)), ((2, 4000), (3, 256))]


@pytest.mark.parametrize('src,out', RESIZE_CASES)
def test_oracle_matches_pillow_resize(src, out):
    Image = pytest.importorskip('PIL.Image')
    image = np.random.RandomState(src[0] * 7 + src[1]).randint(0, 256, size=(*src, 3), dtype=np.uint8)
    want = np.asarray(Image.fromarray(image).resize((out[1], out[0]), Image.BILINEAR))
    assert np.array_equal(ors.resample(image, *out), want)
    top, left = out[0] // 3, out[1] // 4
    oh, ow = out[0] - top, out[1] - left
    assert np.array_equal(ors.resample(image, *out, top, left, oh, ow, 1), want[top:top + oh, left:left + ow][:, ::-1])


def test_identity_axis_coefficients():
    xmin, k = ors.coefficients(17, 17)
    assert np.array_equal(xmin, np.arange(17)) and np.all(k[:, 0] == 1 << 22) and np.all(k[:, 1:] == 0)


def test_fixture_pins_the_draws_and_the_oracle():
    fx = torch.load(os.path.join(HERE, 'golden', 'resample_b200.ptz'), weights_only=False)
    assert [c['seed'] for c in fx['train']] == [t[0] for t in mk.TRAIN]
    for case, (seed, hw, resize) in zip(fx['train'], mk.TRAIN):
        src = mk.make_source(seed, *hw)
        assert np.array_equal(case['source'].numpy(), src.astype(np.uint8))
        torch.manual_seed(seed)
        s = common.Uint8RandomHorizontalFlip(0.5)(common.Uint8RandomResizedCrop(resize)({'image': src, 'label': 0}))
        assert torch.equal(torch.get_rng_state(), case['torch_state']), seed
        top, left, h, w = case['params']
        assert s['resample_geom'].tolist() == [h, w, resize, resize, 0, 0, resize, resize, case['flip']], seed
        assert np.array_equal(s['image'], src[top:top + h, left:left + w].astype(np.uint8))
        assert np.array_equal(ors.apply(s['image'], s['resample_geom']), case['out'].numpy()), seed
    for case in fx['eval']:
        s = common.Uint8CenterCrop(case['crop'])(common.Uint8Resize(case['resize'])(
            {'image': case['source'].numpy().astype(np.float32), 'label': 0}))
        assert np.array_equal(ors.apply(s['image'], s['resample_geom']), case['out'].numpy()), case['seed']


def test_eval_geometry_matches_torchvision():
    T = pytest.importorskip('torchvision.transforms')
    Image = pytest.importorskip('PIL.Image')
    for h, w in [(375, 500), (500, 375), (256, 256), (255, 1000), (1200, 257), (333, 500), (225, 300)]:
        img = Image.new('RGB', (w, h))
        resized = T.Resize(256)(img)
        s = common.Uint8Resize(256)({'image': np.zeros((h, w, 3), np.uint8), 'label': 0})
        assert tuple(s['resample_geom'][2:4]) == (resized.height, resized.width)
        crop_box = T.CenterCrop(224)(resized)
        s = common.Uint8CenterCrop(224)(s)
        top = int(round((resized.height - 224) / 2.0))
        left = int(round((resized.width - 224) / 2.0))
        assert s['resample_geom'].tolist() == [h, w, resized.height, resized.width, top, left, 224, 224, 0]
        assert crop_box.size == (224, 224)


def _ref_modules():
    ref_import = _reference()
    return ref_import.module('SimpleAICV.classification.common'), ref_import.module('SimpleAICV.classification.auto_rand_augment')


def _states():
    return torch.get_rng_state(), random.getstate(), np.random.get_state()


def _same_states(a, b):
    return torch.equal(a[0], b[0]) and a[1] == b[1] and all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))


def _sources(seed, b, classes=10):
    rng = np.random.RandomState(seed)
    sizes = [(int(rng.randint(20, 160)), int(rng.randint(20, 160))) for _ in range(b)]
    return [rng.randint(0, 256, size=(h, w, 3)).astype(np.float32) for h, w in sizes], \
        [int(v) for v in rng.randint(0, classes, size=b)]


def _run(transforms, collate, images, labels):
    return collate([_apply_all(transforms, {'image': im.copy(), 'label': lb}) for im, lb in zip(images, labels)])


def _apply_all(transforms, s):
    for t in transforms:
        s = t(s)
    return s


def _resampled(rs):
    return np.stack([ors.apply(rs.data[o:o + int(g[0]) * int(g[1]) * 3].numpy().reshape(int(g[0]), int(g[1]), 3), g.numpy())
                     for o, g in zip(rs.offsets.tolist(), rs.geom)])


def _normalize(u8, mean, std):
    """The reference's ToTensor + Normalize + permute in float32."""
    x = torch.from_numpy(u8).float().div(255.)
    return ((x - torch.tensor(mean)) / torch.tensor(std)).permute(0, 3, 1, 2)


def test_plain_chain_matches_the_live_reference():
    ref, _ = _ref_modules()
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    for seed in range(30):
        images, labels = _sources(seed, 4)
        torch.manual_seed(seed)
        want = _run([ref.Opencv2PIL(), ref.TorchRandomResizedCrop(resize=48), ref.TorchRandomHorizontalFlip(prob=0.5),
                     ref.TorchMeanStdNormalize(mean=mean, std=std)], ref.ClassificationCollater(), images, labels)
        want_state = _states()
        torch.manual_seed(seed)
        got = _run([common.Uint8RandomResizedCrop(resize=48), common.Uint8RandomHorizontalFlip(prob=0.5)],
                   common.Uint8ClassificationCollater(pin_memory=False), images, labels)
        assert _same_states(_states(), want_state), seed
        assert set(got) == {'label', 'resample'}
        assert torch.equal(_normalize(_resampled(got['resample']), mean, std), want['image']), seed
        assert torch.equal(got['label'], want['label'])


def test_randaugment_mixup_chain_matches_the_live_reference():
    ref, ar = _ref_modules()
    for seed in range(20):
        images, labels = _sources(100 + seed, 4)
        outs = []
        for ours in (False, True):
            torch.manual_seed(seed)
            random.seed(seed)
            np.random.seed(seed)
            if ours:
                tf = [common.Uint8RandomResizedCrop(resize=40), common.Uint8RandomHorizontalFlip(prob=0.5),
                      common.Uint8RandAugment(**mkra.RANDAUG), common.Uint8RandomErasing(**mkmix.ERASE)]
                collate = common.Uint8MixupCutmixClassificationCollater(**mkmix.COLLATE, pin_memory=False)
            else:
                tf = [ref.Opencv2PIL(), ref.TorchRandomResizedCrop(resize=40), ref.TorchRandomHorizontalFlip(prob=0.5),
                      ar.RandAugment(**mkra.RANDAUG), ref.TorchMeanStdNormalize(mean=list(mkmix.MEAN), std=list(mkmix.STD)),
                      ref.RandomErasing(**mkmix.ERASE)]
                collate = ref.MixupCutmixClassificationCollater(**mkmix.COLLATE)
            outs.append((_run(tf, collate, images, labels), _states()))
        (want, want_state), (got, state) = outs
        assert _same_states(state, want_state), seed
        rec = got['mixup']
        resized = _resampled(got['resample'])
        augmented = torch.from_numpy(np.stack([ora.apply(resized[b], rec.randaug_ops[b].numpy(), rec.randaug_f[b].numpy(),
                                                         rec.randaug_affine[b].numpy(), rec.randaug_fill) for b in range(4)]))
        img, soft = omix.apply(augmented, got['label'], rec, mkmix.MEAN, mkmix.STD)
        assert torch.equal(img, want['image'].contiguous()), seed
        assert torch.equal(soft, want['label']), seed


def test_eval_chain_matches_the_live_reference():
    ref, _ = _ref_modules()
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    for seed in range(10):
        images, labels = _sources(200 + seed, 3)
        images = [im for im in images if min(im.shape[:2]) >= 1]
        want = _run([ref.Opencv2PIL(), ref.TorchResize(resize=64), ref.TorchCenterCrop(resize=56),
                     ref.TorchMeanStdNormalize(mean=mean, std=std)], ref.ClassificationCollater(), images, labels)
        got = _run([common.Uint8Resize(64), common.Uint8CenterCrop(56)], common.Uint8ClassificationCollater(pin_memory=False),
                   images, labels)
        assert torch.equal(_normalize(_resampled(got['resample']), mean, std), want['image']), seed


def test_logical_size_follows_the_record():
    """RandAugment's Translate / Rotate and RandomErasing's rectangle use the output size, not the crop's."""
    image = np.random.RandomState(0).randint(0, 256, size=(300, 120, 3)).astype(np.uint8)
    g = np.array([300, 120, 224, 224, 0, 0, 224, 224, 0], np.int32)
    for seed in range(40):
        random.seed(seed)
        np.random.seed(seed)
        s = common.Uint8RandAugment(**mkra.RANDAUG)({'image': image, 'label': 0, 'resample_geom': g.copy()})
        random.seed(seed)
        np.random.seed(seed)
        t = common.Uint8RandAugment(**mkra.RANDAUG)({'image': np.zeros((224, 224, 3), np.uint8), 'label': 0})
        assert np.array_equal(s['randaug_affine'], t['randaug_affine']) and np.array_equal(s['randaug_ops'], t['randaug_ops'])
        np.random.seed(seed)
        e = common.Uint8RandomErasing(prob=1.0)({'image': image, 'label': 0, 'resample_geom': g.copy()})
        np.random.seed(seed)
        f = common.Uint8RandomErasing(prob=1.0)({'image': np.zeros((224, 224, 3), np.uint8), 'label': 0})
        assert np.array_equal(e['erase_rect'], f['erase_rect']) and np.array_equal(e['erase_noise'], f['erase_noise'])


def _geom_samples(sizes, out=(8, 8)):
    rng = np.random.RandomState(1)
    return [{'image': rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8), 'label': i % 3,
             'resample_geom': np.array([h, w, out[0], out[1], 0, 0, out[0], out[1], i % 2], np.int32)}
            for i, (h, w) in enumerate(sizes)]


def test_collaters_pack_ragged_crops():
    samples = _geom_samples([(5, 7), (12, 3), (1, 1), (9, 9)])
    for collate in (common.Uint8ClassificationCollater(pin_memory=False),
                    common.Uint8MixupCutmixClassificationCollater(num_classes=3, pin_memory=False)):
        batch = collate([dict(s) for s in samples])
        assert 'image' not in batch
        rs = batch['resample']
        assert rs.data.dtype == torch.uint8 and rs.data.dim() == 1 and rs.data.numel() == sum(s['image'].size for s in samples)
        assert rs.offsets.dtype == torch.int64 and rs.offsets.tolist() == [0, 105, 213, 216]
        assert rs.geom.dtype == torch.int32 and rs.geom.shape == (4, 9) and rs.out_hw == (8, 8)
        for s, o, g in zip(samples, rs.offsets.tolist(), rs.geom):
            assert np.array_equal(rs.data[o:o + s['image'].size].numpy(), s['image'].reshape(-1))
            assert np.array_equal(g.numpy(), s['resample_geom'])
    assert common.pack_resample([{'image': np.zeros((2, 2, 3), np.uint8), 'label': 0}]) is None


def test_collaters_refuse_mixed_or_mismatched_records():
    samples = _geom_samples([(5, 7), (12, 3)])
    plain = {'image': np.zeros((8, 8, 3), np.uint8), 'label': 0}
    for collate in (common.Uint8ClassificationCollater(pin_memory=False),
                    common.Uint8MixupCutmixClassificationCollater(num_classes=3, pin_memory=False)):
        with pytest.raises(ValueError, match='some samples'):
            collate([samples[0], plain])
        with pytest.raises(ValueError, match='output size'):
            collate(samples[:1] + _geom_samples([(4, 4)], out=(6, 6)))
        bad = dict(samples[1], image=np.zeros((4, 3, 3), np.uint8))
        with pytest.raises(ValueError, match='does not match'):
            collate([samples[0], bad])


@pytest.mark.parametrize('make', [lambda: common.Uint8RandomResizedCrop(224, interpolation='bicubic'),
                                  lambda: common.Uint8RandomResizedCrop(224, ratio=(0.5, 2.0)),
                                  lambda: common.Uint8RandomResizedCrop((224, 200)),
                                  lambda: common.Uint8Resize((256, 256)),
                                  lambda: common.Uint8Resize(256, max_size=300),
                                  lambda: common.Uint8Resize(256, interpolation='nearest'),
                                  lambda: common.Uint8CenterCrop((224, 224))])
def test_unimplemented_options_raise(make):
    with pytest.raises(NotImplementedError, match='shipped'):
        make()


def test_transforms_refuse_out_of_order_or_padding_use():
    with pytest.raises(ValueError, match='would pad'):
        common.Uint8CenterCrop(224)(common.Uint8Resize(200)({'image': np.zeros((300, 400, 3), np.uint8), 'label': 0}))
    with pytest.raises(ValueError, match='no geometry record'):
        common.Uint8CenterCrop(224)({'image': np.zeros((300, 400, 3), np.uint8), 'label': 0})
    with pytest.raises(ValueError, match='no geometry record'):
        common.Uint8RandomHorizontalFlip()({'image': np.zeros((30, 40, 3), np.uint8), 'label': 0})
    with pytest.raises(ValueError, match='already carries'):
        common.Uint8Resize(256)(common.Uint8RandomResizedCrop(224)({'image': np.zeros((30, 40, 3), np.uint8), 'label': 0}))
    with pytest.raises(ValueError, match='expects'):
        common.Uint8RandomResizedCrop(224)({'image': np.zeros((30, 40), np.uint8), 'label': 0})


def test_resample_kernel_sass_has_no_fma_outside_the_divisions():
    """Every float64 operation of u8_resample_kernel is an explicit _rn intrinsic: the only DFMA / FFMA instructions are
    inside the correctly rounded double divisions (their inline sequences between MUFU.RCP64H and the slow-path call, and
    the slow-path subroutines after the kernel's last EXIT)."""
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    lib = os.path.join(ROOT, 'simpleaicv_pytorch_training_examples_b200', 'libsaicv_b200.so')
    if not os.path.exists(cuobjdump) or not os.path.exists(lib):
        pytest.skip('needs cuobjdump and the built library')
    sass = subprocess.run([cuobjdump, '-sass', lib], check=True, capture_output=True, text=True).stdout
    blocks = re.split(r'\n\s*Function : ', sass)
    kernel = [b for b in blocks if b.split('\n', 1)[0].strip().endswith('u8_resample_kernelEPKhPhiiiiNS0_7RsBatchE')]
    assert len(kernel) == 1
    lines = kernel[0].splitlines()
    last_exit = max(i for i, line in enumerate(lines) if re.search(r'\bEXIT\b', line))
    in_division, fused = False, 0
    for i, line in enumerate(lines):
        if 'MUFU.RCP64H' in line:
            in_division = True
        elif 'CALL.REL' in line:
            in_division = False
        if re.search(r'\b(DFMA|FFMA)\b', line):
            assert in_division or i > last_exit, line
            fused += 1
    assert fused > 0 and 'MUFU.RCP64H' in kernel[0]
