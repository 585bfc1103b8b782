"""Oracle: RandAugment(integer=True)'s pixel arithmetic in numpy on CPU, from the draws a sample's RandAugment record
holds (classification.common.Uint8RandAugment).  TEST INFRASTRUCTURE — see oracle/__init__.py.

Restates, for RGB uint8 images, what the reference's 15 increasing-transform ops compute through Pillow
(SimpleAICV/classification/auto_rand_augment.py:50-171 op bodies, :588-605 op set):

- Rotate, ShearX, ShearY, TranslateXRel, TranslateYRel: Image.transform(size, AFFINE, (a, b, c, d, e, f), resample,
  fillcolor).  Output pixel (x, y) reads xin = a (x + 0.5) + b (y + 0.5) + c, yin = d (x + 0.5) + e (y + 0.5) + f in
  float64; outside [0, W) x [0, H) it takes the fill colour.  Otherwise both shift by -0.5, x0 = floor, dx = xin - x0,
  neighbours clamp to the edge.  BILINEAR: v1 = p00 + (p01 - p00) dx, v2 = p10 + (p11 - p10) dx, v = v1 + (v2 - v1) dy,
  truncated.  BICUBIC (4 x 4, along x then along y): p1 = v2, p2 = -v1 + v3, p3 = 2 (v1 - v2) + v3 - v4,
  p4 = -v1 + v2 - v3 + v4, v = p1 + d (p2 + d (p3 + d p4)), clamped to [0, 255] and truncated.  Rotate's coefficients
  are Image.rotate's, computed on the host.
- Brightness, Contrast, Color, Sharpness: Image.blend(degenerate, image, factor) = trunc(clamp(deg + f (img - deg)))
  in float32, f the float64 factor rounded to float32.  Degenerates: zeros; int(mean(L) + 0.5); L per pixel with
  L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16; the SMOOTH filter (3 x 3, weights 1 1 1 / 1 5 1 / 1 1 1 over 13, in
  float32 rows y+1, y, y-1, rounded half up; the border rows and columns are copied).
- AutoContrast, Equalize, Solarize, SolarizeAdd, Posterize, Invert: per-channel 256-entry LUTs (ImageOps), AutoContrast's
  from float64 255 / (hi - lo), Equalize's from the integer histogram steps (clipped at 255).
"""
import numpy as np

(AUTO_CONTRAST, EQUALIZE, INVERT, ROTATE, POSTERIZE, SOLARIZE, SOLARIZE_ADD, COLOR, CONTRAST, BRIGHTNESS, SHARPNESS,
 SHEAR_X, SHEAR_Y, TRANSLATE_X, TRANSLATE_Y) = range(15)
SKIP = -1
BILINEAR, BICUBIC = 2, 3          # PIL.Image.Resampling values
GEOMETRIC = (ROTATE, SHEAR_X, SHEAR_Y, TRANSLATE_X, TRANSLATE_Y)
ENHANCE = (COLOR, CONTRAST, BRIGHTNESS, SHARPNESS)


def luma(img):
    """RGB -> L as Pillow's convert('L'): int64 [H, W]."""
    p = img.astype(np.int64)
    return (p[..., 0] * 19595 + p[..., 1] * 38470 + p[..., 2] * 7471 + 0x8000) >> 16


def smooth(img):
    """ImageFilter.SMOOTH on an RGB image; images narrower or shorter than 3 pixels come back unchanged."""
    h, w = img.shape[:2]
    out = img.copy()
    if h < 3 or w < 3:
        return out
    k1, k5 = np.float32(1) / np.float32(13), np.float32(5) / np.float32(13)
    p = img.astype(np.float32)

    def row(r, kc):
        return (p[r, :-2] * k1 + p[r, 1:-1] * kc) + p[r, 2:] * k1
    ss = np.float32(0) + row(slice(2, None), k1)
    ss = ss + row(slice(1, -1), k5)
    ss = ss + row(slice(0, -2), k1)
    out[1:-1, 1:-1] = np.clip(np.floor(ss.astype(np.float64) + 0.5), 0, 255).astype(np.uint8)
    return out


def blend(deg, img, factor):
    """Image.blend(deg, img, factor) on uint8 RGB in float32."""
    f = np.float32(factor)
    d = deg.astype(np.float32)
    v = d + f * (img.astype(np.float32) - d)
    return np.clip(v, 0, 255).astype(np.uint8)


def lut(img, op, iparam):
    """The op's per-channel LUTs: int64 [3, 256]."""
    i = np.arange(256, dtype=np.int64)
    if op == INVERT:
        return np.tile(255 - i, (3, 1))
    if op == POSTERIZE:
        return np.tile(i & ~(2 ** (8 - iparam) - 1), (3, 1))
    if op == SOLARIZE:
        return np.tile(np.where(i < iparam, i, 255 - i), (3, 1))
    if op == SOLARIZE_ADD:
        return np.tile(np.where(i < 128, np.minimum(255, i + iparam), i), (3, 1))
    out = np.tile(i, (3, 1))
    for c in range(3):
        h = np.bincount(img[..., c].reshape(-1), minlength=256).astype(np.int64)
        nz = np.flatnonzero(h)
        if op == AUTO_CONTRAST:
            lo, hi = int(nz[0]), int(nz[-1])
            if hi > lo:
                scale = 255.0 / (hi - lo)
                offset = -lo * scale
                out[c] = [min(255, max(0, int(x * scale + offset))) for x in range(256)]
        elif op == EQUALIZE:
            if len(nz) > 1:
                step = (int(h.sum()) - int(h[nz[-1]])) // 255
                if step:
                    n = step // 2 + np.concatenate([[0], np.cumsum(h)[:-1]])
                    out[c] = np.minimum(n // step, 255)
    return out


def affine(img, coeffs, resample, fill):
    """Image.transform(size, AFFINE, coeffs, resample, fillcolor=fill) on uint8 RGB."""
    h, w = img.shape[:2]
    a, b, c, d, e, f = (float(v) for v in coeffs)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    xin = a * (xs + 0.5) + b * (ys + 0.5) + c
    yin = d * (xs + 0.5) + e * (ys + 0.5) + f
    inside = (xin >= 0) & (xin < w) & (yin >= 0) & (yin < h)
    xi, yi = np.where(inside, xin, 0.5) - 0.5, np.where(inside, yin, 0.5) - 0.5
    x0, y0 = np.floor(xi).astype(np.int64), np.floor(yi).astype(np.int64)
    dx, dy = (xi - x0)[..., None], (yi - y0)[..., None]
    s = img.astype(np.float64)

    def px(yy, xx):
        return s[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
    if resample == BILINEAR:
        v1 = px(y0, x0) + (px(y0, x0 + 1) - px(y0, x0)) * dx
        v2 = px(y0 + 1, x0) + (px(y0 + 1, x0 + 1) - px(y0 + 1, x0)) * dx
        v = v1 + (v2 - v1) * dy
    elif resample == BICUBIC:
        def cub(v1, v2, v3, v4, t):
            p1, p2 = v2, -v1 + v3
            p3 = 2 * (v1 - v2) + v3 - v4
            p4 = -v1 + v2 - v3 + v4
            return p1 + t * (p2 + t * (p3 + t * p4))
        rows = [cub(*[px(y0 + j, x0 + i) for i in (-1, 0, 1, 2)], dx) for j in (-1, 0, 1, 2)]
        v = cub(*rows, dy)
    else:
        raise ValueError(f'resample {resample}')
    out = np.clip(v, 0, 255).astype(np.uint8)
    out[~inside] = np.asarray(fill, dtype=np.uint8)
    return out


def apply_op(img, op, resample, iparam, factor, coeffs, fill):
    """One layer on uint8 [H, W, 3]; op SKIP returns the image."""
    if op == SKIP:
        return img
    if op in GEOMETRIC:
        return affine(img, coeffs, resample, fill)
    if op in ENHANCE:
        if op == BRIGHTNESS:
            deg = np.zeros_like(img)
        elif op == CONTRAST:
            mean = float(luma(img).sum()) / (img.shape[0] * img.shape[1])
            deg = np.full_like(img, int(mean + 0.5))
        elif op == COLOR:
            deg = np.repeat(luma(img).astype(np.uint8)[..., None], 3, -1)
        else:
            deg = smooth(img)
        return blend(deg, img, factor)
    t = lut(img, op, iparam)
    return np.stack([t[c][img[..., c]] for c in range(3)], -1).astype(np.uint8)


def apply(image_u8, ops, factors, coeffs, fill):
    """One sample: uint8 [H, W, 3] and its record (ops int [L, 4] = (op, resample, iparam, pad), factors float32 [L],
    coeffs float64 [L, 6]) -> uint8 [H, W, 3]."""
    img = np.asarray(image_u8, dtype=np.uint8)
    for layer in range(len(ops)):
        op, resample, iparam = (int(v) for v in np.asarray(ops[layer])[:3])
        img = apply_op(img, op, resample, iparam, np.asarray(factors)[layer], np.asarray(coeffs)[layer], fill)
    return img
