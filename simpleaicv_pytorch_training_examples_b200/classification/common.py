"""Host-side helpers of the classification hot path with the reference's names
(SimpleAICV/classification/common.py:668-685 AverageMeter, :688-709 AccMeter, :843-881 get_amp_type) and the
input-pipeline edge of SURVEY.md 8 f3: ``Uint8ClassificationCollater`` + ``DeviceNormalize`` move the batch over PCIe as
uint8 pixels and normalise on the device; ``Uint8RandomErasing`` + ``Uint8MixupCutmixClassificationCollater`` do the same for
the recipes that end in RandomErasing and Mixup / CutMix, with the random draws on the host and the pixel and label
arithmetic on the device; ``Uint8RandAugment`` makes RandAugment's draws on the host and leaves its pixel arithmetic to the
same device edge; ``Uint8RandomResizedCrop`` / ``Uint8RandomHorizontalFlip`` and ``Uint8Resize`` / ``Uint8CenterCrop``
make torchvision's crop and flip draws on the host and leave the Pillow resize to the device.  The other per-sample
transforms / datasets stay CPU data code (SURVEY.md section 2)."""
import math
import random

import numpy as np
import torch


def load_state_dict(saved_model_path, model, excluded_layer_name=()):
    """classification/common.py:758-800 of the reference: loads the entries of a saved ``state_dict`` file whose name and
    shape match ``model`` (and whose name contains none of ``excluded_layer_name``); an empty path is a no-op."""
    if not saved_model_path:
        return
    saved = torch.load(saved_model_path, map_location=torch.device('cpu'), weights_only=True)
    own = model.state_dict()
    keep = {n: w for n, w in saved.items()
            if n in own and w.shape == own[n].shape and not any(e in n for e in excluded_layer_name)}
    skipped = [n for n in saved if n not in keep]
    if skipped:
        print(f'not loaded: {len(skipped)} of {len(saved)} saved tensors (name / shape mismatch or excluded)')
    model.load_state_dict(keep, strict=False)


class Uint8ClassificationCollater:
    """Counterpart of ClassificationCollater (common.py:645-665) for samples whose 'image' is still the decoder's uint8
    [H, W, 3] array (i.e. the transform list ends BEFORE TorchMeanStdNormalize / Normalize): stacks into ONE pinned uint8
    [B, H, W, 3] tensor (a quarter of the fp32 batch's bytes on the host link) and int64 labels.  ``DeviceNormalize`` (or
    tools.utils.CudaPrefetcher(normalize=...)) finishes the reference's arithmetic on the GPU."""

    def __init__(self, pin_memory=True):
        self.pin_memory = pin_memory

    def __call__(self, data):
        if any('randaug_ops' in s for s in data):
            raise ValueError('samples carry a Uint8RandAugment record, which only Uint8MixupCutmixClassificationCollater '
                             'passes on to the device: this collater would drop it')
        labels = torch.from_numpy(np.array([s['label'] for s in data]).astype(np.float32)).long()
        pin = self.pin_memory and torch.cuda.is_available()
        resample = pack_resample(data, pin)
        if resample is not None:
            return {'label': labels.pin_memory() if pin else labels, 'resample': resample}
        images = np.stack([np.ascontiguousarray(s['image']) for s in data])
        assert images.dtype == np.uint8 and images.ndim == 4 and images.shape[3] == 3, 'expects uint8 [H, W, 3] images'
        images = torch.from_numpy(images)
        if pin:
            images, labels = images.pin_memory(), labels.pin_memory()
        return {'image': images, 'label': labels}


# the int32 geometry record of a Uint8RandomResizedCrop / Uint8Resize sample ('resample_geom') and the rows of
# ResampleBatch.geom: csrc/capi_input.cu's and oracle/resample.py's layout
GEOM_SRC_H, GEOM_SRC_W, GEOM_FULL_H, GEOM_FULL_W, GEOM_TOP, GEOM_LEFT, GEOM_OUT_H, GEOM_OUT_W, GEOM_FLIP = range(9)


class ResampleBatch:
    """The ragged uint8 crops of one batch and their geometry, for the device resize (ops.u8_resample).

    data uint8 [total]: every sample's [src_h, src_w, 3] crop, concatenated (pinned when the collater pins);
    offsets int64 [B]: where image b starts in ``data``; geom int32 [B, 9]: the samples' 'resample_geom' records.  Image b
    is resized to (full_h, full_w) with Pillow's bilinear filter, and the (out_h, out_w) window at (top, left) is kept,
    mirrored when flip is 1."""

    def __init__(self, data, offsets, geom):
        self.data, self.offsets, self.geom = data, offsets, geom

    @property
    def out_hw(self):
        return int(self.geom[0, GEOM_OUT_H]), int(self.geom[0, GEOM_OUT_W])

    def pin_memory(self):
        """Called by DataLoader(pin_memory=True): only the pixels are copied to the device; offsets and geometry are read
        on the host."""
        self.data = self.data.pin_memory()
        return self


def pack_resample(data, pin=False):
    """The samples' crops packed into one ResampleBatch (into pinned memory when ``pin``), or None when no sample carries
    a geometry record.  Raises when only some do, when the output sizes differ or when a crop does not match its record."""
    has = [s.get('resample_geom') is not None for s in data]
    if not any(has):
        return None
    if not all(has):
        raise ValueError('some samples carry a Uint8RandomResizedCrop / Uint8Resize geometry record and some do not')
    geom = np.stack([np.asarray(s['resample_geom'], dtype=np.int32) for s in data])
    if geom.shape[1] != 9 or len({(int(g[GEOM_OUT_H]), int(g[GEOM_OUT_W])) for g in geom}) != 1:
        raise ValueError(f'the samples\' geometry records differ in output size: {sorted({tuple(g[6:8]) for g in geom})}')
    sizes = []
    for s, g in zip(data, geom):
        image = s['image']
        if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.shape != (g[GEOM_SRC_H], g[GEOM_SRC_W], 3):
            raise ValueError(f'a crop of {np.shape(image)} does not match its record\'s source size {tuple(g[:2])}')
        sizes.append(image.size)
    offsets = np.zeros(len(data), dtype=np.int64)
    offsets[1:] = np.cumsum(sizes)[:-1]
    packed = torch.empty(int(sum(sizes)), dtype=torch.uint8, pin_memory=pin)
    flat = packed.numpy()
    for s, off, size in zip(data, offsets, sizes):
        flat[off:off + size] = s['image'].reshape(-1)
    return ResampleBatch(packed, torch.from_numpy(offsets), torch.from_numpy(geom))


def _interpolation_is_bilinear(interpolation):
    return str(getattr(interpolation, 'value', interpolation)).lower() == 'bilinear'


def _source_image(sample, who):
    image = np.asarray(sample['image'])
    if image.ndim != 3 or image.shape[2] != 3 or image.shape[0] < 1 or image.shape[1] < 1:
        raise ValueError(f'{who} expects the decoded [H, W, 3] image, got {image.dtype} {image.shape}')
    if sample.get('resample_geom') is not None:
        raise ValueError(f'{who} starts the transform list: the sample already carries a geometry record')
    return image


def random_resized_crop_params(height, width, scale, ratio):
    """torchvision.transforms.RandomResizedCrop.get_params: the same torch draws from the global generator, in its
    order, -> (top, left, h, w)."""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1]).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,)).item()
            j = torch.randint(0, width - w + 1, size=(1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w = width
        h = height
    return (height - h) // 2, (width - w) // 2, h, w


class Uint8RandomResizedCrop:
    """Takes the place of ``Opencv2PIL(), TorchRandomResizedCrop(resize, scale)`` (SimpleAICV/classification/common.py:
    22-75) in a transform list collated by ``Uint8ClassificationCollater`` or ``Uint8MixupCutmixClassificationCollater``:
    it makes torchvision's crop draws (random_resized_crop_params) and keeps only the crop, as uint8 (np.uint8 of the
    dataset's integer-valued float32 or uint8 image).  The resize to resize x resize is left to the device
    (ops.u8_resample, Pillow's bilinear arithmetic); the sample's 'resample_geom' record holds the crop size, the output
    size, the output window (0, 0, resize, resize) and the flip flag.  Only the shipped setting (bilinear, the default
    ratio) is implemented."""

    def __init__(self, resize=224, scale=(0.08, 1.0), ratio=(3. / 4., 4. / 3.), interpolation='bilinear'):
        if not isinstance(resize, (int, np.integer)):
            raise NotImplementedError(f'Uint8RandomResizedCrop resize={resize!r}: only a square int size (the shipped '
                                      'configs\') is implemented')
        if tuple(ratio) != (3. / 4., 4. / 3.):
            raise NotImplementedError(f'Uint8RandomResizedCrop ratio={ratio!r}: only the default (3/4, 4/3) (the shipped '
                                      'configs\') is implemented')
        if not _interpolation_is_bilinear(interpolation):
            raise NotImplementedError(f'Uint8RandomResizedCrop interpolation={interpolation!r}: only bilinear (the shipped '
                                      'configs\') is implemented')
        self.size, self.scale, self.ratio = int(resize), tuple(scale), tuple(ratio)

    def __call__(self, sample):
        image = _source_image(sample, 'Uint8RandomResizedCrop')
        top, left, h, w = random_resized_crop_params(image.shape[0], image.shape[1], self.scale, self.ratio)
        sample['image'] = image[top:top + h, left:left + w].astype(np.uint8)
        sample['resample_geom'] = np.array([h, w, self.size, self.size, 0, 0, self.size, self.size, 0], dtype=np.int32)
        return sample


class Uint8RandomHorizontalFlip:
    """Takes the place of ``TorchRandomHorizontalFlip(prob)`` after ``Uint8RandomResizedCrop``: torchvision's
    torch.rand(1) < prob draw toggles the record's flip flag; the device mirrors the output."""

    def __init__(self, prob=0.5):
        self.prob = prob

    def __call__(self, sample):
        if sample.get('resample_geom') is None:
            raise ValueError('Uint8RandomHorizontalFlip follows Uint8RandomResizedCrop or Uint8Resize: the sample has no '
                             'geometry record')
        if torch.rand(1) < self.prob:
            sample['resample_geom'][GEOM_FLIP] ^= 1
        return sample


class Uint8Resize:
    """Takes the place of ``Opencv2PIL(), TorchResize(resize)`` (SimpleAICV/classification/common.py:22-37,154-169) in an
    evaluation list: the whole image is kept as uint8 and the record holds torchvision's output size for an int size
    (the short side becomes ``resize``, the long one int(resize * long / short)), which the device resizes to with
    Pillow's bilinear arithmetic.  Only the shipped setting (int size, no max_size, bilinear) is implemented."""

    def __init__(self, resize=256, max_size=None, interpolation='bilinear'):
        if not isinstance(resize, (int, np.integer)):
            raise NotImplementedError(f'Uint8Resize resize={resize!r}: only an int size (the shipped configs\') is '
                                      'implemented')
        if max_size is not None:
            raise NotImplementedError('Uint8Resize max_size: only max_size=None (the shipped configs\') is implemented')
        if not _interpolation_is_bilinear(interpolation):
            raise NotImplementedError(f'Uint8Resize interpolation={interpolation!r}: only bilinear (the shipped '
                                      'configs\') is implemented')
        self.size = int(resize)

    def __call__(self, sample):
        image = _source_image(sample, 'Uint8Resize')
        h, w = image.shape[:2]
        short, long = (w, h) if w <= h else (h, w)
        new_short, new_long = self.size, int(self.size * long / short)
        new_w, new_h = (new_short, new_long) if w <= h else (new_long, new_short)
        sample['image'] = np.ascontiguousarray(image, dtype=np.uint8)
        sample['resample_geom'] = np.array([h, w, new_h, new_w, 0, 0, new_h, new_w, 0], dtype=np.int32)
        return sample


class Uint8CenterCrop:
    """Takes the place of ``TorchCenterCrop(resize)`` after ``Uint8Resize``: the record's output window becomes the
    centred resize x resize square, at torchvision's int(round((H - resize) / 2.0)) / int(round((W - resize) / 2.0)).
    A crop larger than the resized image, which torchvision pads, is refused."""

    def __init__(self, resize=224):
        if not isinstance(resize, (int, np.integer)):
            raise NotImplementedError(f'Uint8CenterCrop resize={resize!r}: only a square int size (the shipped configs\') '
                                      'is implemented')
        self.size = int(resize)

    def __call__(self, sample):
        g = sample.get('resample_geom')
        if g is None:
            raise ValueError('Uint8CenterCrop follows Uint8Resize: the sample has no geometry record')
        h, w = int(g[GEOM_OUT_H]), int(g[GEOM_OUT_W])
        if self.size > h or self.size > w:
            raise ValueError(f'Uint8CenterCrop({self.size}) of a {h} x {w} image would pad, which is not implemented')
        g[GEOM_TOP] += int(round((h - self.size) / 2.0))
        g[GEOM_LEFT] += int(round((w - self.size) / 2.0))
        g[GEOM_OUT_H] = g[GEOM_OUT_W] = self.size
        return sample


def _logical_hw(sample, image):
    """(h, w) of the image a transform sees: the output window of a geometry record, else the array's."""
    g = sample.get('resample_geom')
    return (int(g[GEOM_OUT_H]), int(g[GEOM_OUT_W])) if g is not None else image.shape[:2]


MIX_NONE, MIX_MIXUP, MIX_CUTMIX = 0, 1, 2


class MixupEraseRecord:
    """The host's draws for one batch of ``Uint8MixupCutmixClassificationCollater``; the device applies them
    (ops.u8_mix_erase_normalize, csrc/capi_input.cu).

    rects int32 [B, 4]: (top, left, h, w) of image b's erase rectangle, h = w = 0 when it was not erased;
    offsets int64 [B]: where image b's fp32 [h, w, 3] noise starts in ``noise`` (fp32, the rectangles' noise concatenated);
    mode: MIX_NONE / MIX_MIXUP / MIX_CUTMIX; box: the CutMix box (y0, y1, x0, x1); lam: the (corrected) float64 lambda;
    on_value / off_value: the smoothed one-hot values, computed in float64 as the reference does.

    When the samples came through ``Uint8RandAugment``, its per-sample records are stacked here and applied to the uint8
    images first (ops.u8_rand_augment): randaug_ops int32 [B, L, 4], randaug_f float32 [B, L], randaug_affine float64
    [B, L, 6] and randaug_fill, the (R, G, B) fill colour of the geometric ops; all four are None otherwise."""

    def __init__(self, rects, offsets, noise, mode, box, lam, num_classes, on_value, off_value,
                 randaug_ops=None, randaug_f=None, randaug_affine=None, randaug_fill=None):
        self.rects, self.offsets, self.noise = rects, offsets, noise
        self.mode, self.box, self.lam = mode, box, lam
        self.num_classes, self.on_value, self.off_value = num_classes, on_value, off_value
        self.randaug_ops, self.randaug_f, self.randaug_affine = randaug_ops, randaug_f, randaug_affine
        self.randaug_fill = randaug_fill

    def pin_memory(self):
        """Called by DataLoader(pin_memory=True): the noise and the RandAugment record are copied to the device, the rest
        is read on the host."""
        self.noise = self.noise.pin_memory()
        if self.randaug_ops is not None:
            self.randaug_ops = self.randaug_ops.pin_memory()
            self.randaug_f = self.randaug_f.pin_memory()
            self.randaug_affine = self.randaug_affine.pin_memory()
        return self


# RandAugment(integer=True)'s op set in the reference's order (SimpleAICV/classification/auto_rand_augment.py:588-605):
# the op codes of a Uint8RandAugment record, csrc/capi_input.cu's and oracle/randaugment.py's
RANDAUG_OPS = ('AutoContrast', 'Equalize', 'Invert', 'Rotate', 'PosterizeIncreasing', 'SolarizeIncreasing', 'SolarizeAdd',
               'ColorIncreasing', 'ContrastIncreasing', 'BrightnessIncreasing', 'SharpnessIncreasing', 'ShearX', 'ShearY',
               'TranslateXRel', 'TranslateYRel')
RANDAUG_SKIP = -1
RESAMPLE_BILINEAR, RESAMPLE_BICUBIC = 2, 3   # PIL.Image.Resampling.BILINEAR / BICUBIC, the values random.choice returns


def _randomly_negate(v):
    return -v if random.random() > 0.5 else v


def _rotate_coeffs(degrees, w, h):
    """Image.rotate(degrees) as the AFFINE coefficients Image.transform receives (centre (w / 2, h / 2), no expand);
    a whole turn is the identity, which Pillow returns as a copy."""
    angle = degrees % 360.0
    if angle == 0:
        return (1.0, 0.0, 0.0, 0.0, 1.0, 0.0)
    cx, cy = w / 2, h / 2
    angle = -math.radians(angle)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0,
         round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return tuple(m)


class Uint8RandAugment:
    """Takes the place of ``RandAugment(...)`` (SimpleAICV/classification/auto_rand_augment.py:646-690) in a transform
    list whose batch is collated by ``Uint8MixupCutmixClassificationCollater``: the image stays uint8 [H, W, 3] and the
    draws go into the sample as a record ('randaug_ops', 'randaug_f', 'randaug_affine', 'randaug_fill'); the device
    applies them (ops.u8_rand_augment), bit-identical to the reference's PIL ops.

    The draws are the reference's, in its order: np.random.choice over the 15 ops (with replacement); then per chosen op
    random.random() against prob 0.5, random.gauss(magnitude, magnitude_std) clamped to [0, 10], the level function's
    negate draw (random.random() > 0.5) and, for the five geometric ops, random.choice((BILINEAR, BICUBIC)).  None depends
    on pixel values.  Per layer the record holds int32 (op, resample, iparam, 0) with op = -1 when the prob draw skipped
    it and iparam the Posterize bits, Solarize threshold or SolarizeAdd addend; the float32 enhance factor; and the
    float64 AFFINE coefficients, Rotate's computed as Image.rotate computes them.  Only the shipped setting (integer=True,
    uniform choice, finite magnitude_std, no magnitude_max) is implemented."""

    def __init__(self, magnitude=9, num_layers=2, resize=224, mean=(0.485, 0.456, 0.406), integer=True, weight_idx=None,
                 magnitude_std=0.5, magnitude_max=None):
        if not integer:
            raise NotImplementedError('Uint8RandAugment integer=False: only the increasing op set (the shipped configs\' '
                                      'integer=True) is implemented')
        if weight_idx is not None:
            raise NotImplementedError('Uint8RandAugment weight_idx: only the uniform op choice (the shipped configs\' '
                                      'weight_idx=None) is implemented')
        if magnitude_std == float('inf'):
            raise NotImplementedError('Uint8RandAugment magnitude_std=inf: only a normal magnitude draw (the shipped '
                                      'configs\' magnitude_std=0.5) is implemented')
        if magnitude_max:
            raise NotImplementedError('Uint8RandAugment magnitude_max: only the default bound of 10 (the shipped configs\' '
                                      'magnitude_max=None) is implemented')
        self.magnitude = magnitude
        self.num_layers = num_layers
        self.magnitude_std = float(magnitude_std) if magnitude_std else 0.
        self.fill = tuple(min(255, round(255 * x)) for x in mean)

    def _layer(self, op, w, h):
        """One AugmentOp call's draws (auto_rand_augment.py:338-355) -> (op, resample, iparam, factor, coefficients)."""
        if random.random() > 0.5:
            return RANDAUG_SKIP, 0, 0, 0., (0.,) * 6
        magnitude = self.magnitude
        if self.magnitude_std > 0:
            magnitude = random.gauss(magnitude, self.magnitude_std)
        magnitude = max(0., min(magnitude, 10.))
        name, iparam, factor, coeffs = RANDAUG_OPS[op], 0, 0., (0.,) * 6
        if name == 'Rotate':
            degrees = _randomly_negate((magnitude / 10.) * 30.)
        elif name == 'PosterizeIncreasing':
            iparam = 4 - int((magnitude / 10.) * 4)
        elif name == 'SolarizeIncreasing':
            iparam = 256 - int((magnitude / 10.) * 256)
        elif name == 'SolarizeAdd':
            iparam = int((magnitude / 10.) * 110)
        elif name.endswith('Increasing'):
            factor = max(0.1, 1.0 + _randomly_negate((magnitude / 10.) * .9))
        elif name in ('ShearX', 'ShearY'):
            shear = _randomly_negate((magnitude / 10.) * 0.3)
            coeffs = (1, shear, 0, 0, 1, 0) if name == 'ShearX' else (1, 0, 0, shear, 1, 0)
        elif name in ('TranslateXRel', 'TranslateYRel'):
            pct = _randomly_negate((magnitude / 10.) * 0.45)
            coeffs = (1, 0, pct * w, 0, 1, 0) if name == 'TranslateXRel' else (1, 0, 0, 0, 1, pct * h)
        resample = 0
        if name in ('Rotate', 'ShearX', 'ShearY', 'TranslateXRel', 'TranslateYRel'):
            resample = random.choice((RESAMPLE_BILINEAR, RESAMPLE_BICUBIC))
            if name == 'Rotate':
                coeffs = _rotate_coeffs(degrees, w, h)
        return op, resample, iparam, factor, coeffs

    def __call__(self, sample):
        image = np.asarray(sample['image'])
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f'Uint8RandAugment expects a PIL RGB image or a uint8 [H, W, 3] array, got {image.dtype} {image.shape}')
        h, w = _logical_hw(sample, image)
        chosen = np.random.choice(len(RANDAUG_OPS), self.num_layers, replace=True)
        ops = np.zeros((self.num_layers, 4), dtype=np.int32)
        factors = np.zeros(self.num_layers, dtype=np.float32)
        coeffs = np.zeros((self.num_layers, 6), dtype=np.float64)
        for i, op in enumerate(chosen):
            ops[i, 0], ops[i, 1], ops[i, 2], factors[i], coeffs[i] = self._layer(int(op), w, h)
        sample['image'], sample['randaug_ops'], sample['randaug_f'] = image, ops, factors
        sample['randaug_affine'], sample['randaug_fill'] = coeffs, self.fill
        return sample


class Uint8RandomErasing:
    """Takes the place of ``TorchMeanStdNormalize(mean, std), RandomErasing(...)`` at the end of a transform list
    (SimpleAICV/classification/common.py:228-248,560-642) when the batch is collated by
    ``Uint8MixupCutmixClassificationCollater``: the image stays uint8 [H, W, 3] and the erase rectangle and its noise go
    into the sample ('erase_rect', 'erase_noise') instead of into the pixels.

    The np.random calls are RandomErasing's, in its order: uniform(0, 1) against ``prob``; then up to 10 tries of
    uniform(min_area, max_area), uniform(log aspect range), and, when the rectangle fits, randint(top), randint(left) and
    normal(size=(h, w, 3)).  The noise is kept as float32, the value the reference's assignment into its float32 image
    stores.  Only the shipped setting (mode='pixel', one rectangle) is implemented."""

    def __init__(self, prob=0.25, min_area=0.02, max_area=1 / 3, min_aspect=0.3, max_aspect=None, mode='pixel',
                 min_count=1, max_count=None):
        max_count = max_count if max_count else min_count
        if mode != 'pixel':
            raise NotImplementedError(f"Uint8RandomErasing mode={mode!r}: only mode='pixel' (the shipped configs') is implemented")
        if min_count != 1 or max_count != 1:
            raise NotImplementedError(f'Uint8RandomErasing min_count={min_count}, max_count={max_count}: only one rectangle '
                                      '(the shipped configs\' max_count=1) is implemented')
        self.prob = prob
        self.min_area = min_area
        self.max_area = max_area
        max_aspect = max_aspect if max_aspect else 1 / min_aspect
        self.log_aspect_ratio = (math.log(min_aspect), math.log(max_aspect))

    def __call__(self, sample):
        image = np.asarray(sample['image'])
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f'Uint8RandomErasing expects a PIL RGB image or a uint8 [H, W, 3] array, got {image.dtype} {image.shape}')
        image_h, image_w = _logical_hw(sample, image)
        rect, noise = np.zeros(4, dtype=np.int32), np.zeros(0, dtype=np.float32)
        if np.random.uniform(0, 1) < self.prob:
            area = image_h * image_w
            for _ in range(10):
                target_area = np.random.uniform(self.min_area, self.max_area) * area
                aspect_ratio = math.exp(np.random.uniform(*self.log_aspect_ratio))
                h = int(round(math.sqrt(target_area * aspect_ratio)))
                w = int(round(math.sqrt(target_area / aspect_ratio)))
                if w < image_w and h < image_h:
                    top = np.random.randint(0, image_h - h)
                    left = np.random.randint(0, image_w - w)
                    noise = np.random.normal(loc=0.0, scale=1.0, size=(h, w, 3)).astype(np.float32).reshape(-1)
                    rect[:] = (top, left, h, w)
                    break
        sample['image'], sample['erase_rect'], sample['erase_noise'] = image, rect, noise
        return sample


class Uint8MixupCutmixClassificationCollater:
    """Counterpart of MixupCutmixClassificationCollater (SimpleAICV/classification/mixupcutmixclassificationcollator.py:
    99-284) for samples from ``Uint8RandomErasing`` (or any uint8 [H, W, 3] samples): stacks the images into one pinned
    uint8 [B, H, W, 3] tensor as ``Uint8ClassificationCollater`` does and adds a ``MixupEraseRecord`` under 'mixup'.
    tools.utils.CudaPrefetcher(normalize=(mean, std)) turns the batch into the reference's {'image': fp32 [B, 3, H, W],
    'label': fp32 [B, num_classes]}, bit for bit.

    The batch-mode draws are the reference's, in its order: rand() against mixup_cutmix_prob; with both alphas > 0, rand()
    against switch_to_cutmix_prob; beta(alpha, alpha); for CutMix randint(0, H) for the box centre row and randint(0, W)
    for its column.  The corrected lambda is 1 - box area / (H * W) in float64; when lambda is 1 nothing is mixed.
    Only the shipped setting (use_mixup=True, mode='batch', cutmix_minmax=None) is implemented.

    Samples from ``Uint8RandomResizedCrop`` carry ragged crops: they are packed into a ResampleBatch under 'resample'
    instead of stacked under 'image', and H x W is the records' output size."""

    def __init__(self, use_mixup=True, mixup_alpha=0.8, cutmix_alpha=1.0, cutmix_minmax=None, mixup_cutmix_prob=1.0,
                 switch_to_cutmix_prob=0.5, mode='batch', correct_lam=True, label_smoothing=0.1, num_classes=1000,
                 pin_memory=True):
        if not use_mixup:
            raise NotImplementedError('Uint8MixupCutmixClassificationCollater use_mixup=False: use Uint8ClassificationCollater '
                                      '(the shipped configs use use_mixup=True)')
        if mode != 'batch':
            raise NotImplementedError(f"Uint8MixupCutmixClassificationCollater mode={mode!r}: only mode='batch' (the shipped "
                                      "configs') is implemented")
        if cutmix_minmax is not None:
            raise NotImplementedError('Uint8MixupCutmixClassificationCollater cutmix_minmax: only cutmix_minmax=None (the '
                                      'shipped configs\') is implemented')
        if not (mixup_alpha > 0. or cutmix_alpha > 0.):
            raise ValueError('one of mixup_alpha > 0, cutmix_alpha > 0 must hold')
        self.mixup_alpha = mixup_alpha
        self.cutmix_alpha = cutmix_alpha
        self.mixup_cutmix_prob = mixup_cutmix_prob
        self.switch_to_cutmix_prob = switch_to_cutmix_prob
        self.correct_lam = correct_lam
        self.label_smoothing = label_smoothing
        self.num_classes = num_classes
        self.pin_memory = pin_memory

    def _params_per_batch(self):
        lam, use_cutmix = 1., False
        if np.random.rand() < self.mixup_cutmix_prob:
            if self.mixup_alpha > 0. and self.cutmix_alpha > 0.:
                use_cutmix = np.random.rand() < self.switch_to_cutmix_prob
                alpha = self.cutmix_alpha if use_cutmix else self.mixup_alpha
            elif self.mixup_alpha > 0.:
                alpha = self.mixup_alpha
            else:
                use_cutmix, alpha = True, self.cutmix_alpha
            lam = float(np.random.beta(alpha, alpha))
        return lam, use_cutmix

    def __call__(self, data):
        pin = self.pin_memory and torch.cuda.is_available()
        resample = pack_resample(data, pin)
        if resample is None:
            shape = np.shape(data[0]['image'])
            for s in data:
                img = s['image']
                if np.shape(img) != shape or len(shape) != 3 or shape[2] != 3 or np.asarray(img).dtype != np.uint8:
                    raise ValueError(f'expects uint8 [H, W, 3] images of one shape, got {np.asarray(img).dtype} '
                                     f'{np.shape(img)} next to {shape}')
            h, w = shape[:2]
        else:
            h, w = resample.out_hw
        b = len(data)
        if b % 2 != 0:
            raise ValueError(f'Mixup / CutMix pairs image b with image B-1-b: the batch size must be even (got {b})')
        labels = np.array([s['label'] for s in data]).astype(np.float32).astype(np.int64)
        if labels.min() < 0 or labels.max() >= self.num_classes:
            raise ValueError(f'labels must lie in [0, {self.num_classes}), got {labels.min()}..{labels.max()}')
        rects = np.stack([s.get('erase_rect', np.zeros(4, np.int32)) for s in data]).astype(np.int32)
        noises = [np.asarray(s.get('erase_noise', np.zeros(0, np.float32)), dtype=np.float32).reshape(-1) for s in data]
        offsets = np.zeros(b, dtype=np.int64)
        offsets[1:] = np.cumsum([len(n) for n in noises])[:-1]

        randaug = [s.get('randaug_ops') is not None for s in data]
        if any(randaug) and not all(randaug):
            raise ValueError('some samples carry a Uint8RandAugment record and some do not')
        ra = {}
        if all(randaug):
            if len({tuple(s['randaug_fill']) for s in data}) != 1 or len({np.shape(s['randaug_ops']) for s in data}) != 1:
                raise ValueError('the samples\' Uint8RandAugment records differ in layer count or fill colour')
            ra = dict(randaug_ops=torch.from_numpy(np.stack([s['randaug_ops'] for s in data]).astype(np.int32)),
                      randaug_f=torch.from_numpy(np.stack([s['randaug_f'] for s in data]).astype(np.float32)),
                      randaug_affine=torch.from_numpy(np.stack([s['randaug_affine'] for s in data]).astype(np.float64)),
                      randaug_fill=tuple(int(v) for v in data[0]['randaug_fill']))

        lam, use_cutmix = self._params_per_batch()
        mode, box = MIX_NONE, (0, 0, 0, 0)
        if lam != 1.:
            if use_cutmix:
                ratio = np.sqrt(1 - lam)
                cut_h, cut_w = int(h * ratio), int(w * ratio)
                cy = np.random.randint(0, h)
                cx = np.random.randint(0, w)
                yl, yh = int(np.clip(cy - cut_h // 2, 0, h)), int(np.clip(cy + cut_h // 2, 0, h))
                xl, xh = int(np.clip(cx - cut_w // 2, 0, w)), int(np.clip(cx + cut_w // 2, 0, w))
                if self.correct_lam:
                    lam = 1. - (yh - yl) * (xh - xl) / float(h * w)
                mode, box = MIX_CUTMIX, (yl, yh, xl, xh)
            else:
                mode = MIX_MIXUP
        off_value = self.label_smoothing / self.num_classes
        record = MixupEraseRecord(torch.from_numpy(rects), torch.from_numpy(offsets),
                                  torch.from_numpy(np.concatenate(noises)),
                                  mode, box, lam, self.num_classes, 1. - self.label_smoothing + off_value, off_value, **ra)
        labels = torch.from_numpy(labels)
        if pin:
            labels, record = labels.pin_memory(), record.pin_memory()
        if resample is not None:
            return {'label': labels, 'mixup': record, 'resample': resample}
        images = torch.from_numpy(np.stack([np.ascontiguousarray(s['image']) for s in data]))
        return {'image': images.pin_memory() if pin else images, 'label': labels, 'mixup': record}


class DeviceNormalize:
    """(x / 255 - mean) / std and NHWC -> NCHW on the device (csrc/capi_input.cu): TorchMeanStdNormalize
    (common.py:228-248; mean / std given) or Normalize (:190-206; mean 0, std 1 -> x / 255) followed by the collater's
    permute, bit-identical to the host pipeline.  Raises on CPU tensors: there is no host fallback."""

    def __init__(self, mean=(0., 0., 0.), std=(1., 1., 1.)):
        self.mean, self.std = tuple(float(v) for v in mean), tuple(float(v) for v in std)

    def __call__(self, images_u8, out=None):
        from .. import ops
        if not images_u8.is_cuda:
            raise RuntimeError('DeviceNormalize runs on the GPU (uint8 [B, H, W, 3] device tensor expected)')
        return ops.u8_normalize(images_u8, self.mean, self.std, out=out)


class AverageMeter:
    """Running average (sum of val*n over count)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val, self.avg, self.sum, self.count = 0, 0, 0, 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


class AccMeter:
    """Accumulates top-1 / top-5 correct counts; ``compute()`` fills ``acc1`` / ``acc5`` as fractions."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.acc1_correct_num = 0
        self.acc5_correct_num = 0
        self.sample_num = 0
        self.acc1 = 0
        self.acc5 = 0

    def update(self, acc1_correct_num, acc5_correct_num, sample_num):
        self.acc1_correct_num += acc1_correct_num
        self.acc5_correct_num += acc5_correct_num
        self.sample_num += sample_num

    def compute(self):
        self.acc1 = float(self.acc1_correct_num) / self.sample_num if self.sample_num != 0 else 0
        self.acc5 = float(self.acc5_correct_num) / self.sample_num if self.sample_num != 0 else 0


class SemanticSoftmaxMeter:
    """common.py:712-757 of the reference: accuracy over the semantic tree's levels, counting every (row, level) pair that
    has a label.  compute_per_batch runs one kernel (csrc/capi_loss.cu: first argmax per level, torch.argmax's NaN rule)
    on the SemanticOutputs' full logits and returns (correct, valid) as int64 device scalars: the reference's
    ``result = sum_l mean_valid(correct) * n_valid`` is that integer.  The counts stay on the device until compute()."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.acc1 = 0
        self.sum = 0
        self.count = 0

    def compute_per_batch(self, semantic_outputs, semantic_labels):
        from .. import ops
        from .semantic import SemanticOutputs
        if not isinstance(semantic_outputs, SemanticOutputs):
            raise TypeError('SemanticSoftmaxMeter takes the SemanticOutputs of SemanticTree.convert_outputs_to_semantic_outputs')
        logits = semantic_outputs.logits
        if not logits.is_cuda:
            raise RuntimeError('SemanticSoftmaxMeter runs on H100 kernels only; move the logits to the GPU')
        if logits.dtype not in (torch.float32, torch.bfloat16):
            logits = logits.float()
        t = semantic_outputs.tree.tables(logits.device)
        counts = ops.semantic_accuracy(logits.contiguous(), semantic_labels.long().contiguous(), t.level_cols, t.level_off)
        total = counts.sum(dim=0, dtype=torch.int64)
        return total[0], total[1]

    def update_per_batch(self, result, num_valids_total):
        self.sum += result
        self.count += num_valids_total

    def compute(self):
        count = int(self.count)
        self.acc1 = float(self.sum) / count if count != 0 else 0


def get_amp_type(model):
    """The autocast dtype the reference's loop would select for the device ``model`` lives on.

    Same decision procedure as the reference (compute capability >= 8, torch >= 1.10, CUDA >= 11, device
    name in a whitelist) with 'B200' (and 'B300' / 'GB200') added to the whitelist: the unmodified list
    lacks Blackwell parts, so the reference falls back to fp16 + GradScaler on a B200 (SURVEY.md 0.5).
    The kernels of this package always compute in bf16 with fp32 accumulation; the value is what
    ``train_config`` / the loops report and what a torch-side tail (criterion) may autocast to."""
    device = next(model.parameters()).device
    if device.type != 'cuda':
        return torch.bfloat16
    properties = torch.cuda.get_device_properties(device)
    ok = properties.major >= 8
    ver = tuple(int(v) for v in torch.__version__.split('+')[0].split('.')[:2])
    ok = ok and ver >= (1, 10)
    if torch.version.cuda and float(torch.version.cuda.split('.')[0]) < 11:
        ok = False
    name = torch.cuda.get_device_name(device)
    whitelist = ['RTX PRO 6000', 'H20', 'L20', 'L40', '4090', '5090', 'A100', 'A800', 'H100', 'H800',
                 'B200', 'B300', 'GB200']
    ok = ok and any(n in name for n in whitelist)
    return torch.bfloat16 if ok else torch.float16
