"""Numpy restatement of the float32 image arithmetic of the reference's DETR detection and SAM encoder-distillation input
chains, and of what csrc/capi_input.cu saicv_u8_resize_pad computes on the device:

  translate   cv2.warpAffine(image, [[1, 0, tx], [0, 1, ty]], (w, h)) for a float32 image holding uint8 values
              (SimpleAICV/detection/common.py RandomTranslate): INTER_LINEAR, BORDER_CONSTANT 0.  OpenCV inverts the
              matrix, then fixes each source coordinate to 1/32 pixel (INTER_BITS 5, via a 10-bit AB_SCALE product rounded
              half to even plus a 1/64 rounding offset) and weighs the four taps with products of 1/32 steps.  Every weight
              is a multiple of 1/1024 and every value an integer below 256, so the float32 result is exact: it is the
              integer sum of tap x (32 - f) x ... divided by 1024.
  resize      cv2.resize(image, (out_w, out_h)) INTER_LINEAR for float32 (resizeGeneric, HResizeLinear + VResizeLinear):
              per axis the double scale in / out, the float32 source coordinate (float)((d + 0.5) * scale - 0.5), its
              floor and float32 weights (1 - f, f).  Columns left of the first or right of the last source column take
              that column alone; rows are clamped to the image with their weights kept.  A horizontal pass
              s0 * a0 + s1 * a1, then a vertical pass h0 * b0 + h1 * b1, each product and sum rounded to float32.
  write       the collaters' padded fp32 NCHW batch: DETR's Normalize (x / 255 in float32) and the DETR padding mask,
              or SamNormalize ((x - mean) / std in float64, then stored as float32), the SAM flip mirroring the output
              columns, zeros in the padding.

OpenCV with IPP (the default build of the pip wheel) resizes some ratios with its own arithmetic; this oracle is
OpenCV's own formula, which cv2 follows with cv2.ipp.setUseIPP(False)."""
import numpy as np

INTER_BITS = 5
INTER_TAB_SIZE = 1 << INTER_BITS
AB_BITS = 10
AB_SCALE = 1 << AB_BITS


def translate(image, tx, ty):
    """float32 [h, w, 3] = cv2.warpAffine(float32(image), [[1, 0, tx], [0, 1, ty]], (w, h)) for uint8 image [h, w, 3]."""
    src = np.asarray(image)
    h, w, _ = src.shape
    # the inverse of the translation as warpAffine forms it: [[1, -0, -tx], [-0, 1, -ty]]
    round_delta = AB_SCALE // INTER_TAB_SIZE // 2
    x0 = int(np.rint(-float(tx) * AB_SCALE)) + round_delta
    y0 = np.rint((np.arange(h, dtype=np.float64) + (-float(ty))) * AB_SCALE).astype(np.int64) + round_delta
    X = (x0 + np.arange(w, dtype=np.int64) * AB_SCALE) >> (AB_BITS - INTER_BITS)
    Y = y0 >> (AB_BITS - INTER_BITS)
    sx, fx = X >> INTER_BITS, X & (INTER_TAB_SIZE - 1)
    sy, fy = Y >> INTER_BITS, Y & (INTER_TAB_SIZE - 1)
    pad = np.zeros((h + 2, w + 2, 3), dtype=np.int64)     # one ring of BORDER_CONSTANT zeros around the image
    pad[1:-1, 1:-1] = src

    def tap(dy, dx):
        yy = np.clip(sy + dy + 1, 0, h + 1)[:, None]
        xx = np.clip(sx + dx + 1, 0, w + 1)[None, :]
        return pad[yy, xx]

    wy0, wy1 = (INTER_TAB_SIZE - fy)[:, None, None], fy[:, None, None]
    wx0, wx1 = (INTER_TAB_SIZE - fx)[None, :, None], fx[None, :, None]
    acc = tap(0, 0) * wy0 * wx0 + tap(0, 1) * wy0 * wx1 + tap(1, 0) * wy1 * wx0 + tap(1, 1) * wy1 * wx1
    return (acc.astype(np.float32) * np.float32(1.0 / (INTER_TAB_SIZE * INTER_TAB_SIZE))).astype(np.float32)


def _axis(in_size, out_size):
    """(first tap, second tap, weight of the first, weight of the second) per output index, float32 weights."""
    scale = 1.0 / (out_size / in_size)
    f = ((np.arange(out_size, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def resize(image, out_h, out_w):
    """float32 [out_h, out_w, 3] = cv2.resize(float32 image [h, w, 3], (out_w, out_h)) with OpenCV's INTER_LINEAR formula."""
    src = np.asarray(image, dtype=np.float32)
    h, w, _ = src.shape
    one = np.float32(1.0)
    sx, fx = _axis(w, out_w)
    left, right = sx < 0, sx >= w - 1
    fx[left | right] = 0
    sx = np.where(left, 0, np.where(right, w - 1, sx))
    a0, a1 = (one - fx)[None, :, None], fx[None, :, None]
    s0 = src[:, sx]
    s1 = src[:, np.minimum(sx + 1, w - 1)]
    horiz = s0 * a0 + s1 * a1
    horiz[:, right] = src[:, sx[right]]                  # past the last source column: that column, unweighted
    sy, fy = _axis(h, out_h)
    r0, r1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    b0, b1 = (one - fy)[:, None, None], fy[:, None, None]
    return (horiz[r0] * b0 + horiz[r1] * b1).astype(np.float32)


def resized(image, out_h, out_w, shift=None):
    """The image a sample's record stands for before normalisation: translated when shift = (tx, ty), then resized."""
    src = translate(image, *shift) if shift is not None else np.asarray(image, dtype=np.float32)
    return resize(src, out_h, out_w)


def write_batch(images, size, mean=None, std=None, flips=None, with_mask=False):
    """The collaters' padded batch from resized float32 [h, w, 3] images: fp32 [B, 3, size, size] with x / 255 (mean is
    None) or (x - mean) / std in float64, outputs mirrored where flips[b]; and for DETR the bool [B, size, size] mask,
    True in the padding."""
    n = len(images)
    out = np.zeros((n, size, size, 3), dtype=np.float32)
    mask = np.ones((n, size, size), dtype=bool)
    for b, img in enumerate(images):
        h, w, _ = img.shape
        if flips is not None and flips[b]:
            img = img[:, ::-1]
        if mean is None:
            v = img / np.float32(255.)
        else:
            v = (img.astype(np.float64) - np.asarray(mean, dtype=np.float64)) / np.asarray(std, dtype=np.float64)
        out[b, :h, :w] = v
        mask[b, :h, :w] = False
    out = np.ascontiguousarray(out.transpose(0, 3, 1, 2))
    return (out, mask) if with_mask else out
