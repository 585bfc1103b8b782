"""Tensor-level wrappers over the C ABI: torch is used for device memory and streams only.

Every function launches on torch's current CUDA stream and returns immediately.  Tensors must be
contiguous CUDA tensors; activations are NHWC bf16 (a conv activation of logical shape
[N, C, H, W] is held as a [N, H, W, C] contiguous tensor).
"""
import ctypes

import torch

from . import _lib
from ._lib import ConvShape

EPI_BIAS, EPI_RELU, EPI_RESID, EPI_ADD_BF16, EPI_MUL_DRELU = 1, 2, 16, 32, 512


def _p(t):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), 'saicv ops need contiguous CUDA tensors'
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def conv_out_size(h, pad, r, stride):
    return (h + 2 * pad - r) // stride + 1


def make_conv_shape(n, h, w, c, k, r, s, stride, pad):
    return ConvShape(n, h, w, c, k, r, s, stride, pad)


# ----------------------------------------------------------------------------- dense layers
def gemm_stats_rows(out_rows, out_cols):
    return _lib.load().saicv_gemm_stats_rows(out_rows, out_cols)


def linear_fwd(x, w, bias=None, resid=None, out=None, flags=0, out_f32=False, row_scale=None, rows_per_scale=0,
               stats=None):
    """row_scale: fp32 [M // rows_per_scale] drop-path scale applied to (x w^T + bias) before +resid.
    stats: partial-sum workspace; the epilogue accumulates per-column sum / sum of squares of the
    bf16 output into gemm_stats_rows(M, N) rows of it (hand both to bn_finalize)."""
    M, K = x.shape
    N = w.shape[0]
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.shape[1] == K
    if out is None:
        out = torch.empty(M, N, device=x.device, dtype=torch.float32 if out_f32 else torch.bfloat16)
    _lib.call('saicv_linear_fwd', _p(x), _p(w), _p(bias), _p(resid), _p(row_scale), rows_per_scale, _p(stats),
              _p(out), M, N, K, flags, int(out_f32), _stream())
    return out


def linear_dgrad(dy, w, resid=None, out=None, flags=0, out_f32=False, gelu_pre=None, relu_out=None, add=None):
    """gelu_pre: bf16 [M, K] pre-activation; the result is multiplied by gelu'(gelu_pre) in the epilogue.
    relu_out: bf16 [M, K] ReLU output; the result is zeroed where it is <= 0.  add: bf16 [M, K] added."""
    M, N = dy.shape
    K = w.shape[1]
    assert dy.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.shape[0] == N
    assert (gelu_pre is not None) + (relu_out is not None) + (add is not None) <= 1
    if relu_out is not None:
        gelu_pre, flags = relu_out, flags | EPI_MUL_DRELU
    elif add is not None:
        gelu_pre, flags = add, flags | EPI_ADD_BF16
    if out is None:
        out = torch.empty(M, K, device=dy.device, dtype=torch.float32 if out_f32 else torch.bfloat16)
    _lib.call('saicv_linear_dgrad', _p(dy), _p(w), _p(resid), _p(gelu_pre), _p(out), M, N, K, flags,
              int(out_f32), _stream())
    return out


def wgrad_splits(out_rows, out_cols, reduce_len):
    return _lib.load().saicv_wgrad_splits(out_rows, out_cols, reduce_len)


def wgrad_transposed(out_rows, out_cols):
    """Whether the weight gradient dW [out_rows, out_cols] runs as dW^T on fewer padded tiles (few filters)."""
    return bool(_lib.load().saicv_wgrad_transposed(out_rows, out_cols))


def linear_wgrad(dy, x, partial=None, transposed=False):
    """Returns fp32 partials [splits, N, K] (dW = dy^T x); reduce with reduce_partials.  transposed: partials
    [splits, K, N] of dW^T = x^T dy over the same splits (every element is the same sum)."""
    M, N = dy.shape
    K = x.shape[1]
    splits = wgrad_splits(N, K, M)
    a, b, rows, cols = (x, dy, K, N) if transposed else (dy, x, N, K)
    if partial is None:
        partial = torch.empty(splits, rows, cols, device=dy.device, dtype=torch.float32)
    _lib.call('saicv_linear_wgrad', _p(a), _p(b), _p(partial), M, rows, cols, splits, _stream())
    return partial


def reduce_partials(partial, out, accumulate=False):
    splits = partial.shape[0]
    n = out.numel()
    _lib.call('saicv_reduce_partials', _p(partial), _p(out), splits, n, int(accumulate), _stream())
    return out


# ----------------------------------------------------------------------------- convolutions
def conv_fprop(x, w, cs, out=None, flags=0, stats=None):
    P = conv_out_size(cs.h, cs.pad, cs.r, cs.stride)
    Q = conv_out_size(cs.w, cs.pad, cs.s, cs.stride)
    if out is None:
        out = torch.empty(cs.n, P, Q, cs.k, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_conv_fprop', _p(x), _p(w), _p(stats), _p(out), ctypes.byref(cs), flags, _stream())
    return out


def phase_dgrad_ok(cs):
    """Whether saicv_conv_dgrad takes this stride-2 conv directly (by output phase, on the compact dy): 3x3, pad 1,
    even h and w, w <= 256 (one 128-row tile holds a whole dy row)."""
    return (cs.stride == 2 and cs.r == 3 and cs.s == 3 and cs.pad == 1 and cs.h % 2 == 0 and cs.w % 2 == 0
            and cs.w <= 256)


def conv_dgrad(dy, w, cs, out=None, add=None, mask_bits=None):
    """dy: [n, P, Q, k], the gradient w.r.t. the conv output; cs: the conv's own shape, stride 1 or 2.
    add: optional bf16 [n, h, w, c] tensor summed into the result in the GEMM epilogue.
    mask_bits: optional ReLU mask from bn_apply (needs `add`); the sum is multiplied by it.
    A stride-2 conv that phase_dgrad_ok() rejects, or one with `add`, runs as the stride-1 data gradient of the
    zero-upsampled dy."""
    if cs.stride != 1 and not (phase_dgrad_ok(cs) and add is None and mask_bits is None):
        assert cs.stride == 2, cs.stride
        dy = zero_upsample2(dy, cs.h, cs.w)
        cs = make_conv_shape(cs.n, cs.h, cs.w, cs.c, cs.k, cs.r, cs.s, 1, cs.pad)
    if out is None:
        out = torch.empty(cs.n, cs.h, cs.w, cs.c, device=dy.device, dtype=torch.bfloat16)
    _lib.call('saicv_conv_dgrad', _p(dy), _p(w), _p(add), _p(mask_bits), _p(out), ctypes.byref(cs), _stream())
    return out


def conv_wgrad(dy, x, cs, partial=None):
    P = conv_out_size(cs.h, cs.pad, cs.r, cs.stride)
    Q = conv_out_size(cs.w, cs.pad, cs.s, cs.stride)
    ncols = cs.r * cs.s * cs.c
    splits = wgrad_splits(cs.k, ncols, cs.n * P * Q)
    if partial is None:
        # [splits, k, ncols], or [splits, ncols, k] when saicv_conv_wgrad computes dW^T (few filters)
        shape = (splits, ncols, cs.k) if wgrad_transposed(cs.k, ncols) else (splits, cs.k, ncols)
        partial = torch.empty(shape, device=dy.device, dtype=torch.float32)
    _lib.call('saicv_conv_wgrad', _p(dy), _p(x), _p(partial), ctypes.byref(cs), splits, _stream())
    return partial


ORDER_RSC, ORDER_CRS = 0, 1  # K ordering of weight matrices: implicit GEMM / explicit im2col


def prep_conv_weight(w_f32, out, kpad, order=ORDER_RSC, kp=0, cp=0):
    """kp / cp: padded filter count / channels per tap of `out` (0: unpadded)."""
    k, c, r, s = w_f32.shape
    _lib.call('saicv_prep_conv_weight', _p(w_f32), _p(out), k, c, r, s, kpad, order, kp, cp, _stream())
    return out


def finish_conv_wgrad(partial, grad, kpad, accumulate=False, order=ORDER_RSC, kp=0, cp=0):
    """partial: [splits, kp, kpad], or [splits, kpad, kp] where conv_wgrad / the stem's linear_wgrad computed dW^T
    (wgrad_transposed(kp, kpad); never when kp == kpad)."""
    k, c, r, s = grad.shape
    rows = kp or k
    transposed = tuple(partial.shape[1:]) == (kpad, rows) and wgrad_transposed(rows, kpad)
    _lib.call('saicv_finish_conv_wgrad', _p(partial), _p(grad), partial.shape[0], k, c, r, s, kpad,
              int(accumulate), order, kp, cp, int(transposed), _stream())
    return grad


def cast_bf16(src, out=None):
    if out is None:
        out = torch.empty(src.shape, device=src.device, dtype=torch.bfloat16)
    _lib.call('saicv_cast_bf16', _p(src), _p(out), src.numel(), _stream())
    return out


def u8_normalize(images, mean, std, out=None):
    """images: uint8 [N, H, W, 3] (device) -> fp32 [N, 3, H, W] = (x / 255 - mean[c]) / std[c]: ToTensor + Normalize +
    the collater's permute of the reference (classification/common.py:228-248,645-665) on the device, bit-identical."""
    import ctypes
    assert images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3 and images.is_contiguous()
    n, h, w, _ = images.shape
    if out is None:
        out = torch.empty(n, 3, h, w, device=images.device, dtype=torch.float32)
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    _lib.call('saicv_u8_nhwc_to_nchw_norm', _p(images), _p(out), n, h, w, m3, s3, _stream())
    return out


def u8_mix_erase_normalize(images, labels, mean, std, record, noise, out=None, soft=None):
    """The uint8 edge of the Mixup / CutMix + RandomErasing recipes: images uint8 [N, H, W, 3] and labels int64 [N] (device)
    -> (fp32 [N, 3, H, W], fp32 soft labels [N, num_classes]) as TorchMeanStdNormalize + RandomErasing +
    MixupCutmixClassificationCollater compute them on the host, bit-identical.  record: the batch's
    classification.common.MixupEraseRecord (read on the host); noise: device fp32 whose first record.noise.numel()
    floats hold record.noise."""
    assert images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3 and images.is_contiguous()
    n, h, w, _ = images.shape
    assert labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (n,)
    rects, offsets = record.rects, record.offsets
    assert rects.dtype == torch.int32 and tuple(rects.shape) == (n, 4) and not rects.is_cuda and rects.is_contiguous()
    assert offsets.dtype == torch.int64 and tuple(offsets.shape) == (n,) and not offsets.is_cuda and offsets.is_contiguous()
    used = record.noise.numel()
    assert noise.dtype == torch.float32 and noise.numel() >= used
    if out is None:
        out = torch.empty(n, 3, h, w, device=images.device, dtype=torch.float32)
    if soft is None:
        soft = torch.empty(n, record.num_classes, device=images.device, dtype=torch.float32)
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    box = (ctypes.c_int * 4)(*[int(v) for v in record.box])
    _lib.call('saicv_u8_mix_erase_norm', _p(images), _p(out), n, h, w, m3, s3, ctypes.c_void_p(rects.data_ptr()),
              ctypes.c_void_p(offsets.data_ptr()), _p(noise), used, int(record.mode), box, float(record.lam), _p(labels),
              _p(soft), int(record.num_classes), float(record.on_value), float(record.off_value), _stream())
    return out, soft


def u8_rand_augment(images, record, scratch=None, stats=None):
    """RandAugment(integer=True) applied in place to images uint8 [N, H, W, 3] (device) from the draws the host made:
    record is the batch's classification.common.MixupEraseRecord with its randaug_* fields set (read on the host, and
    copied to the device here).  Bit-identical to the reference's PIL ops.  scratch: device uint8 like images; stats:
    device int32 [N, 770] workspace."""
    assert images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3 and images.is_contiguous()
    n, h, w, _ = images.shape
    ra_ops, ra_f, ra_aff = record.randaug_ops, record.randaug_f, record.randaug_affine
    layers = ra_ops.shape[1]
    assert ra_ops.dtype == torch.int32 and tuple(ra_ops.shape) == (n, layers, 4) and not ra_ops.is_cuda and ra_ops.is_contiguous()
    assert ra_f.dtype == torch.float32 and tuple(ra_f.shape) == (n, layers) and not ra_f.is_cuda and ra_f.is_contiguous()
    assert ra_aff.dtype == torch.float64 and tuple(ra_aff.shape) == (n, layers, 6) and not ra_aff.is_cuda and ra_aff.is_contiguous()
    if scratch is None:
        scratch = torch.empty_like(images)
    assert scratch.dtype == torch.uint8 and scratch.shape == images.shape
    if stats is None:
        stats = torch.empty(n, 770, device=images.device, dtype=torch.int32)
    assert stats.dtype == torch.int32 and stats.numel() >= n * 770
    d_ops, d_f, d_aff = (t.to(images.device, non_blocking=True) for t in (ra_ops, ra_f, ra_aff))
    fill = (ctypes.c_int * 3)(*[int(v) for v in record.randaug_fill])
    _lib.call('saicv_u8_rand_augment', _p(images), _p(scratch), n, h, w, layers, ctypes.c_void_p(ra_ops.data_ptr()),
              ctypes.c_void_p(ra_f.data_ptr()), ctypes.c_void_p(ra_aff.data_ptr()), _p(d_ops), _p(d_f), _p(d_aff), fill,
              _p(stats), _stream())
    return images


def u8_resample(src, offsets, geom, out=None):
    """RandomResizedCrop / Resize + CenterCrop + horizontal flip of torchvision's PIL path on the device, bit-identical:
    src: device uint8 holding the packed [h, w, 3] crops; offsets: host int64 [N] (where image b starts in src); geom: host
    int32 [N, 9] (src_h, src_w, full_h, full_w, top, left, out_h, out_w, flip), the rows of
    classification.common.ResampleBatch.  Returns out uint8 [N, out_h, out_w, 3] (device)."""
    assert src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous()
    n = geom.shape[0]
    assert geom.dtype == torch.int32 and tuple(geom.shape) == (n, 9) and not geom.is_cuda and geom.is_contiguous()
    assert offsets.dtype == torch.int64 and tuple(offsets.shape) == (n,) and not offsets.is_cuda and offsets.is_contiguous()
    oh, ow = (int(v) for v in geom[0, 6:8]) if n else (0, 0)
    if out is None:
        out = torch.empty(n, oh, ow, 3, device=src.device, dtype=torch.uint8)
    assert out.dtype == torch.uint8 and tuple(out.shape) == (n, oh, ow, 3)
    _lib.call('saicv_u8_resample', _p(src), src.numel(), ctypes.c_void_p(offsets.data_ptr()),
              ctypes.c_void_p(geom.data_ptr()), n, _p(out), oh, ow, _stream())
    return out


def u8_resize_pad(src, batch, out=None, mask=None):
    """The DETR / SAM-encoder input batch on the device, bit-identical to oracle/detection_input.py: src is device uint8
    holding batch.data (a detection.common.ResizePadBatch, read on the host for its offsets, geometry, translations and
    normalisation).  Returns out fp32 [N, 3, size, size], and for a batch with ``with_mask`` the bool [N, size, size]
    padding mask (else None)."""
    assert src.is_cuda and src.dtype == torch.uint8 and src.is_contiguous()
    offsets, geom, shift = batch.offsets, batch.geom, batch.shift
    n, size = geom.shape[0], int(batch.size)
    assert geom.dtype == torch.int32 and tuple(geom.shape) == (n, 6) and not geom.is_cuda and geom.is_contiguous()
    assert offsets.dtype == torch.int64 and tuple(offsets.shape) == (n,) and not offsets.is_cuda and offsets.is_contiguous()
    assert shift.dtype == torch.float64 and tuple(shift.shape) == (n, 2) and not shift.is_cuda and shift.is_contiguous()
    if out is None:
        out = torch.empty(n, 3, size, size, device=src.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and tuple(out.shape) == (n, 3, size, size) and out.is_contiguous()
    if batch.with_mask:
        if mask is None:
            mask = torch.empty(n, size, size, device=src.device, dtype=torch.bool)
        assert mask.dtype == torch.bool and tuple(mask.shape) == (n, size, size) and mask.is_contiguous()
    else:
        mask = None
    m3 = s3 = None
    if batch.mean is not None:
        m3 = (ctypes.c_double * 3)(*[float(v) for v in batch.mean])
        s3 = (ctypes.c_double * 3)(*[float(v) for v in batch.std])
    _lib.call('saicv_u8_resize_pad', _p(src), src.numel(), ctypes.c_void_p(offsets.data_ptr()),
              ctypes.c_void_p(geom.data_ptr()), ctypes.c_void_p(shift.data_ptr()), n, size, m3, s3, _p(out), _p(mask),
              _stream())
    return out, mask


def stem_kpad(c, r, s):
    """Columns of the explicit-im2col matrix / weight operand of a c-channel r x s stem conv (filter rows padded to 8,
    total rounded up to the 64-wide reduction block)."""
    return (c * r * ((s + 7) // 8 * 8) + 63) // 64 * 64


def stem_im2col(x, r, s, stride, pad, kpad, out=None):
    n, c, h, w = x.shape
    P, Q = conv_out_size(h, pad, r, stride), conv_out_size(w, pad, s, stride)
    if out is None:
        out = torch.empty(n * P * Q, kpad, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_stem_im2col', _p(x), _p(out), n, c, h, w, r, s, stride, pad, kpad, _stream())
    return out


def zero_upsample2(dy, h, w, out=None):
    n, p, q, c = dy.shape
    if out is None:
        out = torch.empty(n, h, w, c, device=dy.device, dtype=torch.bfloat16)
    _lib.call('saicv_zero_upsample2', _p(dy), _p(out), n, p, q, h, w, c, _stream())
    return out


def add_strided2(dx, dd):
    n, h, w, c = dx.shape
    _, p, q, _ = dd.shape
    _lib.call('saicv_add_strided2', _p(dx), _p(dd), n, p, q, h, w, c, _stream())
    return dx


# ----------------------------------------------------------------------------- batch norm
_WS = {}


def partial_ws(device, ncols):
    """Workspace for the deterministic column reductions (SAICV_BN_PARTIAL_ROWS x ncols floats),
    one per (device, width); safe to share because every use is ordered on the stream."""
    key = (device, ncols)
    ws = _WS.get(key)
    if ws is None:
        ws = _WS[key] = torch.empty(_lib.BN_PARTIAL_ROWS * ncols, device=device, dtype=torch.float32)
    return ws


def bn_stats(y, partials=None):
    """Returns the partial-sum workspace to hand to bn_finalize (same rows, c)."""
    c = y.shape[-1]
    if partials is None:
        partials = partial_ws(y.device, 2 * c)
    _lib.call('saicv_bn_stats', _p(y), _p(partials), y.numel() // c, c, _stream())
    return partials


def bn_finalize(stats, gamma, beta, rmean, rvar, scale_shift, saved, rows, eps, momentum, partial_rows=0):
    """partial_rows: 0 for partials written by bn_stats, else the row count of an epilogue-fused reduction."""
    c = gamma.numel()
    _lib.call('saicv_bn_finalize', _p(stats), partial_rows, _p(gamma), _p(beta), _p(rmean), _p(rvar),
              _p(scale_shift), _p(saved), rows, c, eps, momentum, _stream())


def bn_stats_fold(partials, rows, c, partial_rows=0):
    """The fold of bn_finalize on its own: returns stats fp32 [2 * c + 2] = per-channel sum | sum of squares | the
    row count in two exact parts.  Summed over ranks (an all-reduce), it is what bn_finalize_folded finalizes."""
    stats = torch.empty(2 * c + 2, device=partials.device, dtype=torch.float32)
    _lib.call('saicv_bn_stats_fold', _p(partials), partial_rows, rows, c, _p(stats), _stream())
    return stats


def bn_finalize_folded(stats, gamma, beta, rmean, rvar, scale_shift, saved, eps, momentum):
    """bn_finalize from a bn_stats_fold buffer (all-reduced or not), with the row count it carries."""
    _lib.call('saicv_bn_finalize_folded', _p(stats), _p(gamma), _p(beta), _p(rmean), _p(rvar), _p(scale_shift),
              _p(saved), gamma.numel(), eps, momentum, _stream())


def bn_sync_count(stats, c):
    """The row-count slots of a bn_stats_fold buffer over c channels (the `count` of the synchronized backward)."""
    return stats[2 * c:]


def mask_bits_like(y):
    """Buffer for the packed ReLU mask of an activation [..., C]: int32 [rows, C // 32] (bit j of word w is channel
    32w + j; int32 only because torch has no uint32 arithmetic, the bits are the same)."""
    c = y.shape[-1]
    return torch.empty(y.numel() // c, c // 32, device=y.device, dtype=torch.int32)


def bn_apply(y, scale_shift, out, act, res=None, res_scale_shift=None, mask_bits=None):
    """mask_bits: optional mask_bits_like(y) buffer that receives (out > 0), packed (ReLU only)."""
    c = y.shape[-1]
    _lib.call('saicv_bn_apply', _p(y), _p(scale_shift), _p(res), _p(res_scale_shift), _p(out), _p(mask_bits),
              y.numel() // c, c, act, _stream())
    return out


def bn_bwd_reduce(dout, out, y, saved, sums, act, scale_shift=None, bits=None):
    """Activation mask from `out`, else from the packed ReLU mask `bits`, else recomputed from y with scale_shift."""
    c = y.shape[-1]
    _lib.call('saicv_bn_bwd_reduce', _p(dout), _p(out), _p(bits), _p(y), _p(saved), _p(scale_shift),
              _p(partial_ws(y.device, 2 * c)), _p(sums), y.numel() // c, c, act, _stream())


def bn_bwd_apply(dout, out, y, saved, gamma, sums, dy, dres, dgamma, dbeta, act, accumulate=False,
                 scale_shift=None, bits=None, local_sums=None, count=None):
    """Synchronized BatchNorm: `sums` are the sums reduced over ranks, local_sums this rank's own (for dgamma /
    dbeta) and count = bn_sync_count of the forward's reduced statistics (the global row count)."""
    c = y.shape[-1]
    if local_sums is None and count is None:
        _lib.call('saicv_bn_bwd_apply', _p(dout), _p(out), _p(bits), _p(y), _p(saved), _p(gamma), _p(scale_shift),
                  _p(sums), _p(dy), _p(dres), _p(dgamma), _p(dbeta), y.numel() // c, c, act,
                  int(accumulate), _stream())
    else:
        _lib.call('saicv_bn_bwd_apply_sync', _p(dout), _p(out), _p(bits), _p(y), _p(saved), _p(gamma), _p(scale_shift),
                  _p(sums), _p(local_sums), _p(count), _p(dy), _p(dres), _p(dgamma), _p(dbeta), y.numel() // c, c, act,
                  int(accumulate), _stream())


def bn_bwd_reduce2(g, bits, y_a, y_b, saved_a, saved_b, sums):
    """bn_bwd_reduce of two BatchNorms over the same gradient g (masked by `bits` unless None): sums [4, C] receives
    the [2, C] sums of A then of B, bit-identical to two bn_bwd_reduce calls."""
    c = y_a.shape[-1]
    _lib.call('saicv_bn_bwd_reduce2', _p(g), _p(bits), _p(y_a), _p(y_b), _p(saved_a), _p(saved_b),
              _p(partial_ws(g.device, 4 * c)), _p(sums), y_a.numel() // c, c, _stream())


def bn_bwd_apply2(g, bits, y_a, y_b, saved_a, saved_b, gamma_a, gamma_b, sums, dy_a, dy_b, dgamma_a, dbeta_a,
                  dgamma_b, dbeta_b, accumulate_a=False, accumulate_b=False, local_sums=None, count=None):
    """local_sums / count: as for bn_bwd_apply ([4, C] sums; A and B share the row count)."""
    c = y_a.shape[-1]
    if local_sums is None and count is None:
        _lib.call('saicv_bn_bwd_apply2', _p(g), _p(bits), _p(y_a), _p(y_b), _p(saved_a), _p(saved_b), _p(gamma_a),
                  _p(gamma_b), _p(sums), _p(dy_a), _p(dy_b), _p(dgamma_a), _p(dbeta_a), _p(dgamma_b), _p(dbeta_b),
                  y_a.numel() // c, c, int(accumulate_a), int(accumulate_b), _stream())
    else:
        _lib.call('saicv_bn_bwd_apply2_sync', _p(g), _p(bits), _p(y_a), _p(y_b), _p(saved_a), _p(saved_b), _p(gamma_a),
                  _p(gamma_b), _p(sums), _p(local_sums), _p(count), _p(dy_a), _p(dy_b), _p(dgamma_a), _p(dbeta_a),
                  _p(dgamma_b), _p(dbeta_b), y_a.numel() // c, c, int(accumulate_a), int(accumulate_b), _stream())


def add_bf16(a, b):
    _lib.call('saicv_add_bf16', _p(a), _p(b), a.numel(), _stream())
    return a


# ----------------------------------------------------------------------------- pooling
def maxpool3x3s2_fwd(x, out=None, argmax=None):
    n, h, w, c = x.shape
    P, Q = conv_out_size(h, 1, 3, 2), conv_out_size(w, 1, 3, 2)
    if out is None:
        out = torch.empty(n, P, Q, c, device=x.device, dtype=torch.bfloat16)
    if argmax is None:
        argmax = torch.empty(n, P, Q, c, device=x.device, dtype=torch.uint8)
    _lib.call('saicv_maxpool3x3s2_fwd', _p(x), _p(out), _p(argmax), n, h, w, c, _stream())
    return out, argmax


def maxpool3x3s2_bwd(dy, argmax, h, w, out=None):
    n, _, _, c = dy.shape
    if out is None:
        out = torch.empty(n, h, w, c, device=dy.device, dtype=torch.bfloat16)
    _lib.call('saicv_maxpool3x3s2_bwd', _p(dy), _p(argmax), _p(out), n, h, w, c, _stream())
    return out


def maxpool_fwd(x, k, stride, pad=0, pad_hi=None, oob_zero=False):
    """nn.MaxPool2d(k, stride, pad) on NHWC bf16; pad_hi: padding on the bottom/right edge (defaults to pad);
    oob_zero: padded taps take part with value 0 (ZeroPad2d + unpadded pool) instead of being ignored."""
    n, h, w, c = x.shape
    pad_hi = pad if pad_hi is None else pad_hi
    P, Q = (h + pad + pad_hi - k) // stride + 1, (w + pad + pad_hi - k) // stride + 1
    out = torch.empty(n, P, Q, c, device=x.device, dtype=torch.bfloat16)
    argmax = torch.empty(n, P, Q, c, device=x.device, dtype=torch.uint8)
    _lib.call('saicv_maxpool_fwd', _p(x), _p(out), _p(argmax), n, h, w, c, k, stride, pad, pad_hi, int(oob_zero), _stream())
    return out, argmax


def maxpool_bwd(dy, argmax, h, w, k, stride, pad=0, pad_hi=None):
    n, _, _, c = dy.shape
    pad_hi = pad if pad_hi is None else pad_hi
    out = torch.empty(n, h, w, c, device=dy.device, dtype=torch.bfloat16)
    _lib.call('saicv_maxpool_bwd', _p(dy), _p(argmax), _p(out), n, h, w, c, k, stride, pad, pad_hi, _stream())
    return out


def avgpool_fwd(x, out=None):
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty(n, c, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_avgpool_fwd', _p(x), _p(out), n, h * w, c, _stream())
    return out


def avgpool_bwd(dy, h, w, out=None):
    n, c = dy.shape
    if out is None:
        out = torch.empty(n, h, w, c, device=dy.device, dtype=torch.bfloat16)
    _lib.call('saicv_avgpool_bwd', _p(dy), _p(out), n, h * w, c, _stream())
    return out


def colsum(x, out, accumulate=False):
    c = x.shape[-1]
    is_f32 = x.dtype == torch.float32
    ws = None if is_f32 else partial_ws(x.device, c)
    _lib.call('saicv_colsum', _p(x), _p(ws), _p(out), x.numel() // c, c, int(accumulate), int(is_f32), _stream())
    return out


# ----------------------------------------------------------------------------- masked-token models
def token_gather_fwd(src, idx, fill, pos=None, pos_idx=None, out=None):
    """src fp32 [B, S, C], idx int32 [B, R] (-1 = take `fill` [C]), pos fp32 [P, C] added by row (pos_idx int32 [B, R] or the
    row number): out fp32 [B, R, C] (csrc/capi_tokens.cu)."""
    b, s_rows, c = src.shape
    r = idx.shape[1]
    assert src.dtype == torch.float32 and idx.dtype == torch.int32 and idx.shape[0] == b and src.is_contiguous() and idx.is_contiguous()
    if out is None:
        out = torch.empty(b, r, c, device=src.device, dtype=torch.float32)
    _lib.call('saicv_token_gather_fwd', _p(src), s_rows, _p(idx), _p(fill), _p(pos), _p(pos_idx), _p(out), b, r, c, _stream())
    return out


def token_gather_bwd(dout, idx, src_rows, dsrc_dtype=torch.bfloat16, want_fill=True, zero=True):
    """dout fp32 [B, R, C] -> (dsrc [B, src_rows, C] in `dsrc_dtype`, dfill fp32 [C] or None).  zero: some source rows are
    not referenced by idx (their gradient is 0) - pre-zero dsrc."""
    b, r, c = dout.shape
    assert dout.dtype == torch.float32 and dout.is_contiguous() and dsrc_dtype in (torch.bfloat16, torch.float32)
    dsrc = (torch.zeros if zero else torch.empty)(b, src_rows, c, device=dout.device, dtype=dsrc_dtype)
    part = dfill = None
    if want_fill:
        nslab = _lib.load().saicv_token_fill_slabs(b * r)
        part = torch.empty(nslab, c, device=dout.device, dtype=torch.float32)
    _lib.call('saicv_token_gather_bwd', _p(dout), _p(idx), _p(dsrc), int(dsrc_dtype == torch.bfloat16), src_rows, _p(part), b, r, c, _stream())
    if want_fill:
        dfill = torch.empty(c, device=dout.device, dtype=torch.float32)
        reduce_partials(part, dfill)
    return dsrc, dfill


# ----------------------------------------------------------------------------- ViT blocks
def layernorm_fwd(x, gamma, beta, eps, out=None, stats=None):
    rows, c = x.numel() // x.shape[-1], x.shape[-1]
    assert x.dtype == torch.float32
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    if stats is None:
        stats = torch.empty(2, rows, device=x.device, dtype=torch.float32)
    _lib.call('saicv_layernorm_fwd', _p(x), _p(gamma), _p(beta), _p(out), _p(stats), rows, c, eps, _stream())
    return out, stats


def layernorm_bwd(dy, x, gamma, stats, dgamma, dbeta, dres=None, dx=None, dx_bf16=None, accumulate=False,
                  bf16_row_scale=None, rows_per_scale=0):
    rows, c = x.numel() // x.shape[-1], x.shape[-1]
    assert dy.dtype == torch.bfloat16 and x.dtype == torch.float32
    if dx is None:
        dx = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    _lib.call('saicv_layernorm_bwd', _p(dy), _p(x), _p(gamma), _p(stats), _p(dres), _p(dx), _p(dx_bf16),
              _p(bf16_row_scale), rows_per_scale, _p(partial_ws(x.device, 2 * c)), _p(dgamma), _p(dbeta), rows, c,
              int(accumulate), _stream())
    return dx


def gelu_fwd(u, out=None):
    if out is None:
        out = torch.empty_like(u)
    _lib.call('saicv_gelu_fwd', _p(u), _p(out), u.numel(), _stream())
    return out


def vit_assemble_tokens(patch, cls, pos, b, np_, c, out=None):
    if out is None:
        out = torch.empty(b, np_ + 1, c, device=patch.device, dtype=torch.float32)
    _lib.call('saicv_vit_assemble_tokens', _p(patch), _p(cls), _p(pos), _p(out), b, np_, c, _stream())
    return out


def vit_assemble_tokens_bwd(dx, dpos, dcls, dpatch, accumulate=False):
    b, l, c = dx.shape
    _lib.call('saicv_vit_assemble_tokens_bwd', _p(dx), _p(dpos), _p(dcls), _p(dpatch), b, l - 1, c,
              int(accumulate), _stream())
    return dpatch


def token_pool_fwd(x, mean_pool, out=None):
    b, l, c = x.shape
    if out is None:
        out = torch.empty(b, c, device=x.device, dtype=torch.float32)
    _lib.call('saicv_token_pool_fwd', _p(x), _p(out), b, l, c, int(mean_pool), _stream())
    return out


def token_pool_bwd(dpooled, l, mean_pool, dx=None, dx_bf16=None, bf16_row_scale=None):
    b, c = dpooled.shape
    if dx is None:
        dx = torch.empty(b, l, c, device=dpooled.device, dtype=torch.float32)
    _lib.call('saicv_token_pool_bwd', _p(dpooled), _p(dx), _p(dx_bf16), _p(bf16_row_scale), b, l, c,
              int(mean_pool), _stream())
    return dx


def head_views(x, b, l, h, d):
    """[b, h, l, d] views of the heads packed in the rows of x [b*l, n*h*d] ([b][l][n][h][d]), as attn_fwd / attn_bwd
    take them: q, k, v of a qkv buffer (n = 3), or the one view of an attention output or its gradient (n = 1)."""
    x = x.view(b, l, -1, h, d)
    return tuple(x[:, :, i].permute(0, 2, 1, 3) for i in range(x.shape[2]))


def _bhl_strides(t):
    """Element strides {batch, head, row} of a [B, H, L, D] view whose last dimension is contiguous."""
    assert t.dim() == 4 and t.stride(3) == 1 and t.dtype == torch.bfloat16 and t.is_cuda
    return (ctypes.c_longlong * 3)(t.stride(0), t.stride(1), t.stride(2))


def pack_key_mask(mask, lk):
    """bool [B, Lk] (True = padded key, nn.MultiheadAttention's key_padding_mask) -> int32 bit words
    [B, words] (bit k%32 of word k/32) with words*32 >= lk rounded up to 128."""
    b = mask.shape[0]
    words = (lk + 127) // 128 * 4
    m = torch.zeros(b, words * 32, device=mask.device, dtype=torch.int64)
    m[:, :lk] = mask.to(torch.int64)
    w = (m.view(b, words, 32) << torch.arange(32, device=mask.device)).sum(-1)          # 0 .. 2^32-1
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w)                                         # same bits as int32
    return w.to(torch.int32).contiguous()


def _attn_args(q, k, v, out, lse, scale, mask_bits, dropout_p=0.0, dropout_seed=0, dropout_seed_base=None):
    a = _lib.AttnArgs()
    b, h, lq, dqk = q.shape
    lk, dv = k.shape[2], v.shape[3]
    assert k.shape == (b, h, lk, dqk) and v.shape == (b, h, lk, dv) and out.shape == (b, h, lq, dv)
    a.q, a.k, a.v, a.out, a.lse = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr()
    a.q_strides, a.k_strides, a.v_strides, a.o_strides = _bhl_strides(q), _bhl_strides(k), _bhl_strides(v), _bhl_strides(out)
    a.key_mask_bits = mask_bits.data_ptr() if mask_bits is not None else None
    a.mask_words = mask_bits.shape[1] if mask_bits is not None else 0
    a.b, a.h, a.lq, a.lk, a.dqk, a.dv, a.scale = b, h, lq, lk, dqk, dv, scale
    a.dropout_p, a.dropout_seed = float(dropout_p), int(dropout_seed)
    a.dropout_seed_base = dropout_seed_base.data_ptr() if dropout_seed_base is not None else None
    return a


def attn_fwd(q, k, v, scale, out=None, mask_bits=None, dropout_p=0.0, dropout_seed=0, dropout_seed_base=None):
    """General fused attention.  q [B, H, Lq, Dqk], k [B, H, Lk, Dqk], v [B, H, Lk, Dv]: bf16 VIEWS with a
    contiguous last dimension (any batch / head / row strides).  out: [B, H, Lq, Dv] view to write (default:
    a [B, Lq, H, Dv] buffer viewed as [B, H, Lq, Dv], i.e. heads concatenated per token).  dropout_p > 0: dropout on
    the attention probabilities with the counter-hash mask of dropout_seed (pass the same pair to attn_bwd).
    Returns (out, lse)."""
    b, h, lq, _ = q.shape
    dv = v.shape[3]
    if out is None:
        out = torch.empty(b, lq, h, dv, device=q.device, dtype=torch.bfloat16).permute(0, 2, 1, 3)
    lse = torch.empty(b, h, lq, device=q.device, dtype=torch.float32)
    a = _attn_args(q, k, v, out, lse, scale, mask_bits, dropout_p, dropout_seed, dropout_seed_base)
    _lib.call('saicv_attn_fwd', ctypes.byref(a), _stream())
    return out, lse


def attn_bwd(q, k, v, out, lse, dout, scale, dq, dk, dv, dk_cols=0, mask_bits=None, dropout_p=0.0, dropout_seed=0, dropout_seed_base=None):
    """Gradients of attn_fwd written into the given [B, H, L, D] views dq (Dqk cols), dk (leading dk_cols
    columns; 0 = all) and dv."""
    assert dout.stride() == out.stride(), 'dout must have the layout of out'
    a = _lib.AttnBwdArgs()
    a.fwd = _attn_args(q, k, v, out, lse, scale, mask_bits, dropout_p, dropout_seed, dropout_seed_base)
    delta = torch.empty_like(lse)
    a.dout, a.delta = dout.data_ptr(), delta.data_ptr()
    a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    a.dq_strides, a.dk_strides, a.dv_strides = _bhl_strides(dq), _bhl_strides(dk), _bhl_strides(dv)
    a.dk_cols = dk_cols
    _lib.call('saicv_attn_bwd', ctypes.byref(a), _stream())
    return dq, dk, dv


# ----------------------------------------------------------------------------- VAN kernels
def dwconv_fwd(x, w, bias, k, dil=1, relu=False, flip=False):
    """Depthwise k x k 'same' convolution on NHWC bf16; w fp32 [C, 1, k, k]; flip=True gives the data gradient."""
    n, h, wd, c = x.shape
    out = torch.empty_like(x)
    _lib.call('saicv_dwconv_fwd', _p(x), _p(w), _p(bias), _p(out), n, h, wd, c, k, dil, int(relu), int(flip), _stream())
    return out


def dwconv_dgrad_masked(dy, w, mask, k=7):
    """Data gradient of a k x k depthwise 'same' conv (dilation 1) masked by the ReLU in front of it:
    dwconv^T(dy) * (mask > 0), mask = that ReLU's output (NHWC bf16 like dy)."""
    n, h, wd, c = dy.shape
    assert mask.shape == dy.shape and mask.dtype == torch.bfloat16
    out = torch.empty_like(dy)
    _lib.call('saicv_dwconv_dgrad_masked', _p(dy), _p(w), _p(mask), _p(out), n, h, wd, c, k, _stream())
    return out


def avgpool_stream_fwd(x):
    """x: NHWC stream [n, h, w, c] (bf16 or fp32) -> bf16 [n, c] mean over h*w, summed in fp32."""
    n, h, w, c = x.shape
    out = torch.empty(n, c, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_avgpool_stream_fwd', _p(x), int(x.dtype == torch.float32), _p(out), n, h * w, c, _stream())
    return out


def avgpool_stream_bwd(dy, h, w, dx_f32=True):
    """dy bf16 [n, c] -> [n, h, w, c] = dy / (h*w), fp32 (or bf16)."""
    n, c = dy.shape
    assert dy.dtype == torch.bfloat16
    out = torch.empty(n, h, w, c, device=dy.device, dtype=torch.float32 if dx_f32 else torch.bfloat16)
    _lib.call('saicv_avgpool_stream_bwd', _p(dy), _p(out), int(dx_f32), n, h * w, c, _stream())
    return out


def dwconv_wgrad(dy, x, dw, k, dil=1, accumulate=False):
    n, h, wd, c = x.shape
    nblk = _lib.load().saicv_dwconv_wgrad_blocks(n * h * wd)
    partial = torch.empty(nblk * k * k * c, device=x.device, dtype=torch.float32)
    _lib.call('saicv_dwconv_wgrad', _p(dy), _p(x), _p(partial), _p(dw), n, h, wd, c, k, dil, int(accumulate), _stream())
    return dw


def mul_bf16(a, b):
    out = torch.empty_like(a)
    _lib.call('saicv_mul_bf16', _p(a), _p(b), _p(out), a.numel(), _stream())
    return out


def gate_bwd(dg, c1, dlk, p1):
    out = torch.empty_like(dg)
    _lib.call('saicv_gate_bwd', _p(dg), _p(c1), _p(dlk), _p(p1), _p(out), dg.numel(), _stream())
    return out


def ls_residual_fwd(x, branch, shortcut, ls, row_scale=None, rows_per_scale=0):
    c = x.shape[-1]
    rows = x.numel() // c
    out = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    _lib.call('saicv_ls_residual_fwd', _p(x), int(x.dtype == torch.float32), _p(branch), _p(shortcut), _p(ls), _p(row_scale),
              rows_per_scale, _p(out), rows, c, _stream())
    return out


def ls_residual_bwd(dxn, branch, shortcut, ls, dls, accumulate=False, row_scale=None, rows_per_scale=0):
    c = dxn.shape[-1]
    rows = dxn.numel() // c
    dy = torch.empty(dxn.shape, device=dxn.device, dtype=torch.bfloat16)
    _lib.call('saicv_ls_residual_bwd', _p(dxn), _p(branch), _p(shortcut), _p(ls), _p(row_scale), rows_per_scale, _p(dy),
              _p(partial_ws(dxn.device, 2 * c)), _p(dls), rows, c, int(accumulate), _stream())
    return dy


def bn_stats_generic(x):
    """Partial sums for bn_finalize (pass partial_rows=bn_generic_rows(rows, c))."""
    c = x.shape[-1]
    rows = x.numel() // c
    partial = partial_ws(x.device, 2 * c)
    _lib.call('saicv_bn_stats_generic', _p(x), int(x.dtype == torch.float32), _p(partial), rows, c, _stream())
    return partial, _lib.load().saicv_bn_generic_partial_rows(rows, c)


def bn_apply_generic(x, scale_shift, out_f32):
    c = x.shape[-1]
    out = torch.empty(x.shape, device=x.device, dtype=torch.float32 if out_f32 else torch.bfloat16)
    _lib.call('saicv_bn_apply_generic', _p(x), int(x.dtype == torch.float32), _p(scale_shift), _p(out), int(out_f32),
              x.numel() // c, c, _stream())
    return out


def bn_bwd_generic(x, g, saved, gamma, dgamma, dbeta, dres=None, dx_f32=True, accumulate=False):
    c = x.shape[-1]
    rows = x.numel() // c
    dx = torch.empty(x.shape, device=x.device, dtype=torch.float32 if dx_f32 else torch.bfloat16)
    sums = torch.empty(2 * c, device=x.device, dtype=torch.float32)
    _lib.call('saicv_bn_bwd_generic', _p(x), int(x.dtype == torch.float32), _p(g), int(g.dtype == torch.float32), _p(saved),
              _p(gamma), _p(dres), _p(partial_ws(x.device, 2 * c)), _p(sums), _p(dx), int(dx_f32), _p(dgamma), _p(dbeta),
              rows, c, int(accumulate), _stream())
    return dx


def bn_bwd_generic_reduce(x, g, saved):
    """The reduce half of bn_bwd_generic: returns sums fp32 [2 * C] (sum g | sum g * xhat)."""
    c = x.shape[-1]
    sums = torch.empty(2 * c, device=x.device, dtype=torch.float32)
    _lib.call('saicv_bn_bwd_generic_reduce', _p(x), int(x.dtype == torch.float32), _p(g), int(g.dtype == torch.float32),
              _p(saved), _p(partial_ws(x.device, 2 * c)), _p(sums), x.numel() // c, c, _stream())
    return sums


def bn_bwd_generic_apply(x, g, saved, gamma, sums, dgamma, dbeta, dres=None, dx_f32=True, accumulate=False,
                         local_sums=None, count=None):
    """The apply half of bn_bwd_generic; local_sums / count as for bn_bwd_apply.  Returns dx."""
    c = x.shape[-1]
    dx = torch.empty(x.shape, device=x.device, dtype=torch.float32 if dx_f32 else torch.bfloat16)
    _lib.call('saicv_bn_bwd_generic_apply', _p(x), int(x.dtype == torch.float32), _p(g), int(g.dtype == torch.float32),
              _p(saved), _p(gamma), _p(dres), _p(sums), _p(local_sums), _p(count), _p(dx), int(dx_f32), _p(dgamma),
              _p(dbeta), x.numel() // c, c, int(accumulate), _stream())
    return dx


def im2col_nhwc(x, k, stride, pad):
    n, h, w, c = x.shape
    P, Q = conv_out_size(h, pad, k, stride), conv_out_size(w, pad, k, stride)
    cols = torch.empty(n * P * Q, k * k * c, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_im2col_nhwc', _p(x), _p(cols), n, h, w, c, k, stride, pad, _stream())
    return cols, P, Q


def col2im_nhwc(dcols, n, h, w, c, k, stride, pad):
    dx = torch.empty(n, h, w, c, device=dcols.device, dtype=torch.bfloat16)
    _lib.call('saicv_col2im_nhwc', _p(dcols), _p(dx), n, h, w, c, k, stride, pad, _stream())
    return dx


# ----------------------------------------------------------------------------- SAM image encoder kernels
def window_partition(x, ws):
    """x bf16 [B, H, W, C] -> (windows [B*nW, ws*ws, C], (nwy, nwx)); padding tokens are zero."""
    b, h, w, c = x.shape
    nwy, nwx = (h + ws - 1) // ws, (w + ws - 1) // ws
    out = torch.empty(b * nwy * nwx, ws * ws, c, device=x.device, dtype=torch.bfloat16)
    _lib.call('saicv_window_partition', _p(x), _p(out), b, h, w, c, ws, _stream())
    return out, (nwy, nwx)


def window_unpartition(windows, b, h, w, ws):
    c = windows.shape[-1]
    out = torch.empty(b, h, w, c, device=windows.device, dtype=torch.bfloat16)
    _lib.call('saicv_window_unpartition', _p(windows), _p(out), b, h, w, c, ws, _stream())
    return out


def add_pos_embed(x, pos):
    """x fp32 (any shape holding B copies of pos' extent) += pos fp32, broadcast over the batch, in place."""
    assert x.numel() % pos.numel() == 0
    _lib.call('saicv_add_pos_embed', _p(x), _p(pos), x.numel() // pos.numel(), pos.numel(), _stream())
    return x


def relpos_dqk(hd, sh, sw):
    return (hd + sh + sw + 15) // 16 * 16


def relpos_nip(sh, sw):
    return (2 * sh - 1 + 2 * sw - 1 + 63) // 64 * 64


def relpos_build(qkv, rel_pos_h, rel_pos_w, bw, heads, hd, sh, sw, scale, aux=None):
    """qkv bf16 [bw, sh*sw, 3*heads*hd] -> (qe, ke) bf16 [bw, heads, sh*sw, dqk] for attn_fwd(scale=1): the decomposed
    rel-pos bias q . R_h[qh - kh] + q . R_w[qw - kw] as extra score columns.  The dot products are ONE GEMM of the
    tensor-core engine (T = qc rtab^T); `aux` (a dict) receives qc and rtab for relpos_bwd."""
    dqk, nip = relpos_dqk(hd, sh, sw), relpos_nip(sh, sw)
    rows = bw * heads * sh * sw
    dev = qkv.device
    qc = torch.empty(rows, hd, device=dev, dtype=torch.bfloat16)
    _lib.call('saicv_relpos_pack_q', _p(qkv), _p(qc), bw, heads, hd, sh * sw, _stream())
    rtab = torch.empty(nip, hd, device=dev, dtype=torch.bfloat16)
    _lib.call('saicv_relpos_table', _p(rel_pos_h), _p(rel_pos_w), _p(rtab), sh, sw, nip, hd, _stream())
    t = linear_fwd(qc, rtab)                                   # [rows, nip] bf16
    qe = torch.empty(bw, heads, sh * sw, dqk, device=dev, dtype=torch.bfloat16)
    ke = torch.empty_like(qe)
    _lib.call('saicv_relpos_gather', _p(qkv), _p(t), _p(qe), _p(ke), bw, heads, hd, sh, sw, dqk, nip, scale, _stream())
    if aux is not None:
        aux['qc'], aux['rtab'] = qc, rtab
    return qe, ke


def relpos_bwd(dqe, qkv, rel_pos_h, rel_pos_w, dqkv, d_rel_pos_h, d_rel_pos_w, bw, heads, hd, sh, sw, scale, accumulate=False, aux=None):
    """From the score-operand gradient dqe: dq into the q slot of dqkv and the gradients of the two rel-pos tables.  Both
    are GEMMs of the tensor-core engine on the re-indexed bias-column gradients ef (include/saicv_b200.h):
    dq = scale * dqe[:, :hd] + ef rtab,  [d rel_pos_h ; d rel_pos_w] = ef^T qc."""
    dqk, nip = dqe.shape[-1], relpos_nip(sh, sw)
    rows = bw * heads * sh * sw
    nh, nw = 2 * sh - 1, 2 * sw - 1
    dev = dqe.device
    if aux is not None and 'qc' in aux:
        qc, rtab = aux['qc'], aux['rtab']
    else:
        qc = torch.empty(rows, hd, device=dev, dtype=torch.bfloat16)
        _lib.call('saicv_relpos_pack_q', _p(qkv), _p(qc), bw, heads, hd, sh * sw, _stream())
        rtab = torch.empty(nip, hd, device=dev, dtype=torch.bfloat16)
        _lib.call('saicv_relpos_table', _p(rel_pos_h), _p(rel_pos_w), _p(rtab), sh, sw, nip, hd, _stream())
    ef = torch.empty(rows, nip, device=dev, dtype=torch.bfloat16)
    _lib.call('saicv_relpos_shift', _p(dqe), _p(ef), bw, heads, hd, sh, sw, dqk, nip, _stream())
    dqx = linear_dgrad(ef, rtab, out_f32=True)                 # [rows, hd] fp32
    _lib.call('saicv_relpos_dq_combine', _p(dqe), _p(dqx), _p(dqkv), bw, heads, hd, sh * sw, dqk, scale, _stream())
    part = linear_wgrad(ef, qc)                                # [splits, nip, hd]
    tables = torch.empty(nip, hd, device=dev, dtype=torch.float32)
    reduce_partials(part, tables)
    reduce_partials(tables[:nh].view(1, nh, hd), d_rel_pos_h, accumulate=accumulate)
    reduce_partials(tables[nh:nh + nw].view(1, nw, hd), d_rel_pos_w, accumulate=accumulate)


# ----------------------------------------------------------------------------- DETR transformer glue
def postln_fwd(z, gamma, beta, eps, pos=None, want_y=True, want_yb=True, want_ypb=False, yb_out=None):
    """Post-LN of the fp32 stream: returns (y fp32 | None, yb bf16 | None, ypb bf16(y + pos[row % pos_rows]) | None, stats).
    yb_out: bf16 [rows, c] buffer to receive yb."""
    rows, c = z.shape
    assert z.dtype == torch.float32
    y = torch.empty_like(z) if want_y else None
    yb = yb_out if yb_out is not None else (torch.empty(rows, c, device=z.device, dtype=torch.bfloat16) if want_yb else None)
    ypb = torch.empty(rows, c, device=z.device, dtype=torch.bfloat16) if want_ypb else None
    stats = torch.empty(2, rows, device=z.device, dtype=torch.float32)
    _lib.call('saicv_postln_fwd', _p(z), _p(gamma), _p(beta), eps, _p(y), _p(yb), _p(pos), pos.shape[0] if pos is not None else 0,
              _p(ypb), _p(stats), rows, c, _stream())
    return y, yb, ypb, stats


def postln_bwd(dy, z, gamma, stats, dgamma, dbeta, dres=None, want_dz=True, want_dzb=True, accumulate=False):
    rows, c = z.shape
    assert dy.dtype == torch.float32 and z.dtype == torch.float32
    dz = torch.empty_like(z) if want_dz else None
    dzb = torch.empty(rows, c, device=z.device, dtype=torch.bfloat16) if want_dzb else None
    _lib.call('saicv_postln_bwd', _p(dy), _p(z), _p(gamma), _p(stats), _p(dres), _p(dz), _p(dzb), _p(partial_ws(z.device, 2 * c)),
              _p(dgamma), _p(dbeta), rows, c, int(accumulate), _stream())
    return dz, dzb


def add_pos_cast(x, pos=None, want_xb=True, want_xpb=True):
    rows, c = x.shape
    xb = torch.empty(rows, c, device=x.device, dtype=torch.bfloat16) if want_xb else None
    xpb = torch.empty(rows, c, device=x.device, dtype=torch.bfloat16) if (want_xpb and pos is not None) else None
    _lib.call('saicv_add_pos_cast', _p(x), _p(pos), pos.shape[0] if pos is not None else 0, _p(xb), _p(xpb), rows, c, _stream())
    return xb, xpb


def dropout(x, p, seed, resid=None, out_f32=None, out=None, row_scale=None, elems_per_scale=0, seed_base=None):
    """out = (keep ? x / (1 - p) : 0) * row_scale[index // elems_per_scale] (+ resid); counter-hash mask
    (csrc/dropout_hash.cuh), same seed => same mask.  seed_base: int64 device tensor [1] added to `seed` on the device
    (graph-safe: a captured step refreshes it every replay)."""
    if out_f32 is None:
        out_f32 = x.dtype == torch.float32 or resid is not None
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float32 if out_f32 else torch.bfloat16)
    _lib.call('saicv_dropout', _p(x), int(x.dtype == torch.float32), _p(resid), _p(row_scale), elems_per_scale, _p(out), int(out_f32),
              x.numel(), float(p), int(seed), _p(seed_base), _stream())
    return out


def heads_pack(src, col0, b, l, h, hd, dp, scale=1.0, extra=None, extra_const=0.0):
    """src bf16 [b*l, ld] -> [b, h, l, dp]: head columns scaled, column hd = extra[b*l] (or the constant), rest 0."""
    dst = torch.empty(b, h, l, dp, device=src.device, dtype=torch.bfloat16)
    _lib.call('saicv_heads_pack', _p(src), src.shape[1], col0, _p(extra), float(extra_const), _p(dst), b, l, h, hd, dp, float(scale), _stream())
    return dst


def heads_unpack(src, dst, col0, hd, scale=1.0):
    """src bf16 [b, h, l, dp] -> dst bf16 [b*l, ld] columns col0 .. col0 + h*hd (the leading hd columns of every head, scaled)."""
    b, h, l, dp = src.shape
    _lib.call('saicv_heads_unpack', _p(src), _p(dst), dst.shape[1], col0, b, l, h, hd, dp, float(scale), _stream())
    return dst


def detr_decode(logits, boxes, scaled_sizes, num_classes, min_score, topn, max_objects):
    """logits fp32 / bf16 [B, Q, classes + 1], boxes fp32 [B, Q, 4] (cxcywh in [0, 1]), scaled_sizes fp32 [B, 2] (h, w)
    -> fp32 [B, max_objects, 6] rows {score, class, x1, y1, x2, y2}, padded with {-1, -1, 0, 0, 0, 0}
    (include/saicv_b200.h saicv_detr_decode)."""
    b, q, k = logits.shape
    assert logits.dtype in (torch.float32, torch.bfloat16) and boxes.dtype == torch.float32 and tuple(boxes.shape) == (b, q, 4)
    assert scaled_sizes.dtype == torch.float32 and tuple(scaled_sizes.shape) == (b, 2)
    out = torch.empty(b, max_objects, 6, device=logits.device, dtype=torch.float32)
    _lib.call('saicv_detr_decode', _p(logits), int(logits.dtype == torch.bfloat16), _p(boxes), _p(scaled_sizes), _p(out), b, q, k,
              num_classes, float(min_score), topn, max_objects, _stream())
    return out


# ----------------------------------------------------------------------------- SAMLoss
def sam_loss_sums(logits, targets, alpha, gamma, mask_threshold):
    """logits fp32 / bf16 [B, M, H, W], targets fp32 [B, 1, H, W] -> fp32 [B, M, 6] per-mask sums (include/saicv_b200.h)."""
    b, m = logits.shape[:2]
    n = logits[0, 0].numel()
    assert logits.is_contiguous() and targets.is_contiguous() and targets.dtype == torch.float32 and targets.numel() == b * n
    part = torch.empty(_lib.load().saicv_sam_loss_partial_floats(b, m, n), device=logits.device, dtype=torch.float32)
    sums = torch.empty(b, m, 6, device=logits.device, dtype=torch.float32)
    _lib.call('saicv_sam_loss_sums', _p(logits), int(logits.dtype == torch.bfloat16), _p(targets), _p(part), _p(sums), b, m, n,
              float(alpha), float(gamma), float(mask_threshold), _stream())
    return sums


def sam_loss_bwd(logits, targets, coef, alpha, gamma):
    """Gradient of the loss w.r.t. the mask logits (dtype of logits) from the per-mask coefficients coef fp32 [B, M, 3]."""
    b, m = logits.shape[:2]
    n = logits[0, 0].numel()
    dl = torch.empty_like(logits)
    _lib.call('saicv_sam_loss_bwd', _p(logits), int(logits.dtype == torch.bfloat16), _p(targets), _p(coef.contiguous()), _p(dl),
              int(logits.dtype == torch.bfloat16), b, m, n, float(alpha), float(gamma), _stream())
    return dl


# ----------------------------------------------------------------------------- SemanticSoftmaxLoss
def semantic_softmax_fwd(logits, labels, level_cols, level_off, factors, smoothing):
    """logits fp32 / bf16 [B, N], semantic labels int64 [B, L], level tables int32 (include/saicv_b200.h), factors fp32 [L]
    -> (loss fp32 [], lse fp32 [B, L])."""
    b, n = logits.shape
    levels = labels.shape[1]
    assert labels.dtype == torch.int64 and labels.shape[0] == b and factors.dtype == torch.float32 and factors.numel() >= levels
    lse = torch.empty(b, levels, device=logits.device, dtype=torch.float32)
    terms = torch.empty(b, levels, device=logits.device, dtype=torch.float32)
    loss = torch.empty((), device=logits.device, dtype=torch.float32)
    _lib.call('saicv_semantic_softmax_fwd', _p(logits), int(logits.dtype == torch.bfloat16), _p(labels), _p(level_cols), _p(level_off),
              _p(factors), _p(lse), _p(terms), _p(loss), b, n, levels, float(smoothing), _stream())
    return loss, lse


def semantic_softmax_bwd(logits, labels, col_level, level_cols, level_off, factors, lse, grad, smoothing):
    """Gradient fp32 [B, N] of grad (fp32 device scalar) * loss w.r.t. the logits."""
    b, n = logits.shape
    dl = torch.empty(b, n, device=logits.device, dtype=torch.float32)
    _lib.call('saicv_semantic_softmax_bwd', _p(logits), int(logits.dtype == torch.bfloat16), _p(labels), _p(col_level), _p(level_cols),
              _p(level_off), _p(factors), _p(lse), _p(grad), _p(dl), b, n, labels.shape[1], float(smoothing), _stream())
    return dl


def semantic_accuracy(logits, labels, level_cols, level_off):
    """int32 [L, 2]: per level, rows whose first argmax over the level's columns equals the label, and rows with a label."""
    b, n = logits.shape
    levels = labels.shape[1]
    assert labels.dtype == torch.int64 and labels.shape[0] == b
    counts = torch.empty(levels, 2, device=logits.device, dtype=torch.int32)
    _lib.call('saicv_semantic_accuracy', _p(logits), int(logits.dtype == torch.bfloat16), _p(labels), _p(level_cols), _p(level_off),
              _p(counts), b, n, levels, _stream())
    return counts


# ----------------------------------------------------------------------------- DINOv3 kernels
def rope_qk(qkv, sin, cos, b, l, heads, hd, backward=False):
    """In place on the q and k slices of packed qkv bf16 [b*l, 3*heads*hd]: the rotary embedding with the fp32 table
    sin / cos [l, hd] (backward=True: its transpose, applied to dq / dk of a dqkv buffer)."""
    assert qkv.dtype == torch.bfloat16 and qkv.shape == (b * l, 3 * heads * hd)
    assert sin.dtype == cos.dtype == torch.float32 and sin.shape == cos.shape == (l, hd)
    _lib.call('saicv_rope_qk_bwd' if backward else 'saicv_rope_qk_fwd', _p(qkv), _p(sin), _p(cos), b, l, heads, hd, _stream())
    return qkv


def swiglu_fwd(a, b, out=None):
    """h = silu(a) * b (bf16)."""
    assert a.dtype == b.dtype == torch.bfloat16 and a.shape == b.shape
    if out is None:
        out = torch.empty_like(a)
    _lib.call('saicv_swiglu_fwd', _p(a), _p(b), _p(out), a.numel(), _stream())
    return out


def swiglu_bwd(dh, a, b):
    """Returns (da, db) of h = silu(a) * b."""
    assert dh.dtype == a.dtype == b.dtype == torch.bfloat16 and dh.shape == a.shape == b.shape
    da, db = torch.empty_like(a), torch.empty_like(b)
    _lib.call('saicv_swiglu_bwd', _p(dh), _p(a), _p(b), _p(da), _p(db), a.numel(), _stream())
    return da, db
