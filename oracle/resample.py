"""Numpy restatement of Pillow's bilinear Image.resize for 8-bit images (Resample.c ImagingResample, PRECISION_BITS 22)
with the output window and the horizontal flip of a classification.common geometry record: what torchvision's PIL path
computes for RandomResizedCrop + RandomHorizontalFlip and for Resize + CenterCrop, and what csrc/capi_input.cu
saicv_u8_resample computes on the device.

Per axis, output index xx of an in_size -> out_size resize takes the source taps [xmin, xmin + n) with float64
triangle weights normalised by their sum and rounded to 22-bit fixed point.  The horizontal pass runs first and rounds
to uint8; the vertical pass runs over those values with the same rounding.  An axis that keeps its size gets the
weights [2^22, 0], the identity Pillow reaches by skipping the pass."""
import numpy as np

PRECISION_BITS = 22


def _triangle(x):
    x = -x if x < 0.0 else x
    return 1.0 - x if x < 1.0 else 0.0


def coefficients(in_size, out_size):
    """(xmin int64 [out_size], k int64 [out_size, ksize]) of Pillow's precompute_coeffs + normalize_coeffs_8bpc."""
    scale = in_size / out_size
    support = max(scale, 1.0)
    ss = 1.0 / support
    ksize = int(np.ceil(support)) * 2 + 1
    xmins = np.zeros(out_size, dtype=np.int64)
    k = np.zeros((out_size, ksize), dtype=np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size)
        w = [_triangle((x + xmin - center + 0.5) * ss) for x in range(xmax - xmin)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            if ww != 0.0:
                v = v / ww
            k[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        xmins[xx] = xmin
    return xmins, k


def _clip8(acc):
    return np.where(acc >= (1 << PRECISION_BITS << 8), 255, np.where(acc <= 0, 0, acc >> PRECISION_BITS)).astype(np.uint8)


def _pass(src, in_size, out_size, first, count, axis):
    """One pass along ``axis`` (1: columns, 0: rows) of uint8 [H, W, 3] ``src`` for output indices [first, first + count)."""
    xmin, k = coefficients(in_size, out_size)
    xmin, k = xmin[first:first + count], k[first:first + count]
    acc = np.full(src.shape[:axis] + (count,) + src.shape[axis + 1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for j in range(k.shape[1]):
        idx = np.minimum(xmin + j, in_size - 1)           # taps past n have weight 0
        taps = np.take(src, idx, axis=axis).astype(np.int64)
        weight = k[:, j].reshape((1, count, 1) if axis == 1 else (count, 1, 1))
        acc += taps * weight
    return _clip8(acc)


def resample(image, full_h, full_w, top=0, left=0, out_h=None, out_w=None, flip=0):
    """uint8 [H, W, 3] -> the (out_h, out_w) window at (top, left) of its bilinear resize to (full_h, full_w), mirrored
    when ``flip``: Image.resize((full_w, full_h), BILINEAR), then crop, then FLIP_LEFT_RIGHT."""
    image = np.ascontiguousarray(image, dtype=np.uint8)
    h, w = image.shape[:2]
    out_h = full_h if out_h is None else out_h
    out_w = full_w if out_w is None else out_w
    tmp = _pass(image, w, full_w, left, out_w, axis=1)
    out = _pass(tmp, h, full_h, top, out_h, axis=0)
    return np.ascontiguousarray(out[:, ::-1]) if flip else out


def apply(image, geom):
    """The output of one sample from its crop and its int32 [9] geometry record (classification.common GEOM_*)."""
    g = [int(v) for v in geom]
    assert image.shape[:2] == (g[0], g[1]), (image.shape, g)
    return resample(image, g[2], g[3], g[4], g[5], g[6], g[7], g[8])
