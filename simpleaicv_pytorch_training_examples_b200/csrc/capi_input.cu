// Input-pipeline edge (SURVEY.md 8 f3): the batch crosses PCIe as the uint8 HWC pixels the decoder produced and is
// normalised on the device, instead of as fp32 tensors normalised per sample on the host
// (SimpleAICV/classification/common.py:228-248 TorchMeanStdNormalize = ToTensor + Normalize, then
// ClassificationCollater :645-665 stacks [B, H, W, 3] fp32 and permutes to [B, 3, H, W]; tools/scripts.py:143 `.cuda()`).
//
//   out[b][c][h][w] = (float(in[b][h][w][c]) / 255 - mean[c]) / std[c]          fp32 NCHW, the models' input contract
//
// with IEEE divisions in the reference's order (ToTensor: x.float().div(255); Normalize: sub_(mean).div_(std)), so the
// result is bit-identical to the host pipeline.  HBM-bound: 3 B/pixel read + 12 B/pixel written; the host->device copy
// shrinks 4x (38.5 MB instead of 154 MB for a 256 x 224^2 batch).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"

namespace saicv {
namespace {

constexpr int kInThreads = 256;

struct Norm3 {
  float mean[3], std[3];
};

__device__ __forceinline__ float norm1(uint32_t u, float mean, float std) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(u), 255.0f), mean), std);
}

// one thread = 4 consecutive pixels of one image (12 bytes in, one float4 per channel plane out); hw % 4 == 0
__global__ void __launch_bounds__(kInThreads)
u8_nhwc_to_nchw_norm_vec_kernel(const uint32_t* __restrict__ in, float* __restrict__ out, long long groups, int hw4, Norm3 nm) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < groups; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hw4;
    const int g = (int)(i - b * hw4);
    const uint32_t w0 = __ldg(in + i * 3), w1 = __ldg(in + i * 3 + 1), w2 = __ldg(in + i * 3 + 2);
    // bytes: p0 = {w0[0..2]}, p1 = {w0[3], w1[0..1]}, p2 = {w1[2..3], w2[0]}, p3 = {w2[1..3]}
    const uint32_t px[4][3] = {{w0 & 255u, (w0 >> 8) & 255u, (w0 >> 16) & 255u},
                               {w0 >> 24, w1 & 255u, (w1 >> 8) & 255u},
                               {(w1 >> 16) & 255u, w1 >> 24, w2 & 255u},
                               {(w2 >> 8) & 255u, (w2 >> 16) & 255u, w2 >> 24}};
    float* o = out + (b * 3) * (long long)hw4 * 4 + (long long)g * 4;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      *reinterpret_cast<float4*>(o + (long long)c * hw4 * 4) =
          make_float4(norm1(px[0][c], nm.mean[c], nm.std[c]), norm1(px[1][c], nm.mean[c], nm.std[c]),
                      norm1(px[2][c], nm.mean[c], nm.std[c]), norm1(px[3][c], nm.mean[c], nm.std[c]));
  }
}

__global__ void __launch_bounds__(kInThreads)
u8_nhwc_to_nchw_norm_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, long long pixels, long long hw, Norm3 nm) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pixels; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hw, r = i - b * hw;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[(b * 3 + c) * hw + r] = norm1(in[i * 3 + c], nm.mean[c], nm.std[c]);
  }
}

// ---- Mixup / CutMix + RandomErasing(mode='pixel') on the uint8 edge ---------------------------------------------------
// The reference's train tail for the ImageNet recipes with soft labels (classification/common.py:597-642 RandomErasing
// after TorchMeanStdNormalize, mixupcutmixclassificationcollator.py:140-167,269-284 batch-mode MixupCutmixClassification-
// Collater) as one pass: every output pixel depends on the same pixel of image b and of its partner n-1-b only, so one
// thread owns the pair and each input byte is read once.  The random draws were made on the host; they arrive as the
// per-image erase rectangles (with their fp32 noise) and one (mode, box, lam) for the batch.
constexpr int kMixMaxImages = 1024;   // per launch: the rectangle table travels in the kernel's parameter space

struct MixErase {
  int4 rect[kMixMaxImages];            // top, left, h, w; h == 0 or w == 0: not erased
  long long noise_off[kMixMaxImages];  // offset of image b's [h][w][3] noise in `noise`
};

struct MixArgs {
  Norm3 nm;
  const float* noise;
  int mode;                            // 0: no mix, 1: mixup, 2: cutmix
  int y0, y1, x0, x1;                  // cutmix box [y0, y1) x [x0, x1)
  float lam, lam1;                     // (float)lam, (float)(1 - lam)
};

// the image's value after TorchMeanStdNormalize + RandomErasing: the stored noise inside the rectangle, else norm1
__device__ __forceinline__ float erased_or_norm(uint32_t u, int c, int y, int x, const int4& r, long long off,
                                                const MixArgs& a) {
  if ((unsigned)(y - r.x) < (unsigned)r.z && (unsigned)(x - r.y) < (unsigned)r.w)
    return __ldg(a.noise + off + ((long long)(y - r.x) * r.w + (x - r.y)) * 3 + c);
  return norm1(u, a.nm.mean[c], a.nm.std[c]);
}

// out[b] and out[n-1-b] from v(b) = va and v(n-1-b) = vb; mixup as fmul, fmul, fadd (torch's mul_ / add_ on the host)
__device__ __forceinline__ void mix_pair(float va, float vb, int y, int x, const MixArgs& a, float& oa, float& ob) {
  if (a.mode == 1) {
    oa = __fadd_rn(__fmul_rn(va, a.lam), __fmul_rn(vb, a.lam1));
    ob = __fadd_rn(__fmul_rn(vb, a.lam), __fmul_rn(va, a.lam1));
  } else if (a.mode == 2 && y >= a.y0 && y < a.y1 && x >= a.x0 && x < a.x1) {
    oa = vb;
    ob = va;
  } else {
    oa = va;
    ob = vb;
  }
}

__device__ __forceinline__ void unpack4(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t (&px)[4][3]) {
  px[0][0] = w0 & 255u; px[0][1] = (w0 >> 8) & 255u; px[0][2] = (w0 >> 16) & 255u;
  px[1][0] = w0 >> 24; px[1][1] = w1 & 255u; px[1][2] = (w1 >> 8) & 255u;
  px[2][0] = (w1 >> 16) & 255u; px[2][1] = w1 >> 24; px[2][2] = w2 & 255u;
  px[3][0] = (w2 >> 8) & 255u; px[3][1] = (w2 >> 16) & 255u; px[3][2] = w2 >> 24;
}

// one thread = 4 consecutive pixels of image p and of image n-1-p; hw % 4 == 0
__global__ void __launch_bounds__(kInThreads)
u8_mix_erase_norm_vec_kernel(const uint32_t* __restrict__ in, float* __restrict__ out, long long groups, int n, int hw4, int w,
                             MixArgs a, const __grid_constant__ MixErase er) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < groups; i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i / hw4), q = n - 1 - p;
    const int g = (int)(i - (long long)p * hw4);
    const uint32_t* ip = in + ((long long)p * hw4 + g) * 3;
    const uint32_t* iq = in + ((long long)q * hw4 + g) * 3;
    uint32_t pa[4][3], pb[4][3];
    unpack4(__ldg(ip), __ldg(ip + 1), __ldg(ip + 2), pa);
    unpack4(__ldg(iq), __ldg(iq + 1), __ldg(iq + 2), pb);
    const int4 ra = er.rect[p], rb = er.rect[q];
    const long long offa = er.noise_off[p], offb = er.noise_off[q];
    float oa[3][4], ob[3][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = g * 4 + k, y = r / w, x = r - y * w;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        mix_pair(erased_or_norm(pa[k][c], c, y, x, ra, offa, a), erased_or_norm(pb[k][c], c, y, x, rb, offb, a), y, x, a,
                 oa[c][k], ob[c][k]);
    }
    float* op = out + (long long)p * 3 * hw4 * 4 + (long long)g * 4;
    float* oq = out + (long long)q * 3 * hw4 * 4 + (long long)g * 4;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      *reinterpret_cast<float4*>(op + (long long)c * hw4 * 4) = make_float4(oa[c][0], oa[c][1], oa[c][2], oa[c][3]);
      *reinterpret_cast<float4*>(oq + (long long)c * hw4 * 4) = make_float4(ob[c][0], ob[c][1], ob[c][2], ob[c][3]);
    }
  }
}

// one thread = one pixel of image p and of image n-1-p (any h, w)
__global__ void __launch_bounds__(kInThreads)
u8_mix_erase_norm_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, long long pairs_px, int n, long long hw, int w,
                         MixArgs a, const __grid_constant__ MixErase er) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs_px; i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i / hw), q = n - 1 - p;
    const long long r = i - (long long)p * hw;
    const int y = (int)(r / w), x = (int)(r - (long long)y * w);
    const int4 ra = er.rect[p], rb = er.rect[q];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float oa, ob;
      mix_pair(erased_or_norm(in[((long long)p * hw + r) * 3 + c], c, y, x, ra, er.noise_off[p], a),
               erased_or_norm(in[((long long)q * hw + r) * 3 + c], c, y, x, rb, er.noise_off[q], a), y, x, a, oa, ob);
      out[((long long)p * 3 + c) * hw + r] = oa;
      out[((long long)q * 3 + c) * hw + r] = ob;
    }
  }
}

// soft[b][j] = fadd(fmul(y1, lam), fmul(y2, 1 - lam)), y1 / y2 the smoothed one-hots of labels[b] / labels[n-1-b]
// (mixupcutmixclassificationcollator.py:13-31 one_hot + mixup_label)
__global__ void __launch_bounds__(kInThreads)
mix_soft_label_kernel(const long long* __restrict__ labels, float* __restrict__ soft, int n, int classes, float on, float off,
                      float lam, float lam1) {
  const long long total = (long long)n * classes;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / classes), j = (int)(i - (long long)b * classes);
    const float y1 = __ldg(labels + b) == j ? on : off, y2 = __ldg(labels + (n - 1 - b)) == j ? on : off;
    soft[i] = __fadd_rn(__fmul_rn(y1, lam), __fmul_rn(y2, lam1));
  }
}

}  // namespace
}  // namespace saicv

using namespace saicv;

extern "C" int saicv_u8_mix_erase_norm(const void* in, float* out, int n, int h, int w, const float* mean3, const float* std3,
                                       const int* rects, const long long* noise_off, const float* noise, long long noise_len,
                                       int mode, const int* box4, double lam, const long long* labels, float* soft,
                                       int num_classes, float on_value, float off_value, void* stream) {
  const char* fn = "saicv_u8_mix_erase_norm";
  if (!in || !out || !labels || !soft || !rects || !noise_off) return set_error("%s: null pointer", fn);
  if (n < 2 || n % 2 != 0 || n > kMixMaxImages)
    return set_error("%s: the batch must be even, 2 <= n <= %d (n=%d)", fn, kMixMaxImages, n);
  if (h <= 0 || w <= 0 || num_classes <= 0) return set_error("%s: empty image or class count (h=%d w=%d classes=%d)", fn, h, w, num_classes);
  if (mode < 0 || mode > 2) return set_error("%s: mode %d is not 0 (none), 1 (mixup) or 2 (cutmix)", fn, mode);
  if (!isfinite(lam)) return set_error("%s: lam is not finite", fn);
  MixArgs a;
  for (int c = 0; c < 3; ++c) {
    a.nm.mean[c] = mean3[c];
    a.nm.std[c] = std3[c];
  }
  a.noise = noise;
  a.mode = mode;
  a.y0 = a.y1 = a.x0 = a.x1 = 0;
  if (mode == 2) {
    if (!box4) return set_error("%s: cutmix needs a box", fn);
    a.y0 = box4[0], a.y1 = box4[1], a.x0 = box4[2], a.x1 = box4[3];
    if (a.y0 < 0 || a.y0 > a.y1 || a.y1 > h || a.x0 < 0 || a.x0 > a.x1 || a.x1 > w)
      return set_error("%s: cutmix box [%d, %d) x [%d, %d) outside the %d x %d image", fn, a.y0, a.y1, a.x0, a.x1, h, w);
  }
  a.lam = (float)lam;
  a.lam1 = (float)(1.0 - lam);
  static thread_local MixErase er;
  for (int b = 0; b < n; ++b) {
    const int top = rects[4 * b], left = rects[4 * b + 1], rh = rects[4 * b + 2], rw = rects[4 * b + 3];
    const long long off = noise_off[b];
    if (top < 0 || left < 0 || rh < 0 || rw < 0)
      return set_error("%s: image %d has a negative erase rectangle (%d, %d, %d, %d)", fn, b, top, left, rh, rw);
    if (rh > 0 && rw > 0) {
      if ((long long)top + rh > h || (long long)left + rw > w)
        return set_error("%s: image %d's erase rectangle (top %d, left %d, %d x %d) leaves the %d x %d image", fn, b, top, left, rh, rw, h, w);
      if (!noise || off < 0 || off > noise_len || (long long)rh * rw * 3 > noise_len - off)
        return set_error("%s: image %d's noise [%lld, %lld) is past the buffer of %lld floats", fn, b, off,
                         off + (long long)rh * rw * 3, noise_len);
    }
    er.rect[b] = make_int4(top, left, rh, rw);
    er.noise_off[b] = off;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long hw = (long long)h * w, pairs = n / 2;
  if (hw % 4 == 0 && ((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 15) == 0) {
    const long long groups = pairs * (hw / 4);
    u8_mix_erase_norm_vec_kernel<<<grid_1d(groups, kInThreads), kInThreads, 0, st>>>(reinterpret_cast<const uint32_t*>(in), out, groups, n,
                                                                          (int)(hw / 4), w, a, er);
    if (check_launch("u8_mix_erase_norm_vec_kernel")) return 1;
  } else {
    u8_mix_erase_norm_kernel<<<grid_1d(pairs * hw, kInThreads), kInThreads, 0, st>>>(reinterpret_cast<const uint8_t*>(in), out, pairs * hw, n,
                                                                         hw, w, a, er);
    if (check_launch("u8_mix_erase_norm_kernel")) return 1;
  }
  mix_soft_label_kernel<<<grid_1d((long long)n * num_classes, kInThreads), kInThreads, 0, st>>>(labels, soft, n, num_classes, on_value,
                                                                                     off_value, a.lam, a.lam1);
  return check_launch("mix_soft_label_kernel");
}

extern "C" int saicv_u8_nhwc_to_nchw_norm(const void* in, float* out, int n, int h, int w, const float* mean3,
                                          const float* std3, void* stream) {
  if (n <= 0 || h <= 0 || w <= 0) return set_error("saicv_u8_nhwc_to_nchw_norm: empty batch");
  Norm3 nm;
  for (int c = 0; c < 3; ++c) {
    nm.mean[c] = mean3[c];
    nm.std[c] = std3[c];
  }
  const long long hw = (long long)h * w, pixels = hw * n;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (hw % 4 == 0 && ((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 15) == 0) {
    const long long groups = pixels / 4;
    u8_nhwc_to_nchw_norm_vec_kernel<<<grid_1d(groups, kInThreads), kInThreads, 0, st>>>(reinterpret_cast<const uint32_t*>(in), out, groups, (int)(hw / 4), nm);
    return check_launch("u8_nhwc_to_nchw_norm_vec_kernel");
  }
  u8_nhwc_to_nchw_norm_kernel<<<grid_1d(pixels, kInThreads), kInThreads, 0, st>>>(reinterpret_cast<const uint8_t*>(in), out, pixels, hw, nm);
  return check_launch("u8_nhwc_to_nchw_norm_kernel");
}
