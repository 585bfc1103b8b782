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

#include <algorithm>

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

// ---- RandAugment(integer=True) on the uint8 edge -----------------------------------------------------------------------
// The reference's RandAugment (classification/auto_rand_augment.py:646-690) runs two of 15 PIL ops per image.  The host
// made every draw (classification.common.Uint8RandAugment); per image and layer the record holds (op, resample, iparam),
// the enhance factor and the AFFINE coefficients.  Per layer a stats pass takes the histograms / luma sum the op needs,
// then one pass writes every output pixel with Pillow's arithmetic: integer LUTs, float32 blends, float64 affine gathers.
// Every float operation is an explicit _rn intrinsic so that nothing contracts into an FMA Pillow does not execute.
constexpr int kRAMaxImages = 1024;   // per launch: the stats list travels in the kernel's parameter space
constexpr int kRAMaxLayers = 16;
constexpr int kRAStatsWords = 770;   // per image: 3 x 256 histogram bins, then the 64-bit luma sum
constexpr int kRAPixelsPerThread = 8;

enum RAOp {
  kRASkip = -1, kAutoContrast, kEqualize, kInvert, kRotate, kPosterize, kSolarize, kSolarizeAdd, kColor, kContrast,
  kBrightness, kSharpness, kShearX, kShearY, kTranslateX, kTranslateY, kRANumOps
};
constexpr int kBilinear = 2, kBicubic = 3;   // PIL.Image.Resampling values

__host__ __device__ __forceinline__ bool ra_geometric(int op) {
  return op == kRotate || op == kShearX || op == kShearY || op == kTranslateX || op == kTranslateY;
}
__host__ __device__ __forceinline__ bool ra_enhance(int op) { return op >= kColor && op <= kSharpness; }
__host__ __device__ __forceinline__ bool ra_lut(int op) { return op >= kAutoContrast && op <= kSolarizeAdd && op != kRotate; }
__host__ __device__ __forceinline__ bool ra_needs_stats(int op) {
  return op == kAutoContrast || op == kEqualize || op == kContrast;
}

struct RAStatsList {
  int count;
  unsigned short img[kRAMaxImages];
};

// Pillow's RGB -> L (Convert.c rgb2l)
__device__ __forceinline__ uint32_t ra_luma(uint32_t r, uint32_t g, uint32_t b) {
  return (r * 19595u + g * 38470u + b * 7471u + 0x8000u) >> 16;
}

// per listed image: 3 x 256 channel histograms (AutoContrast, Equalize) or the sum of L (Contrast), with integer atomics
__global__ void __launch_bounds__(kInThreads)
ra_stats_kernel(const uint8_t* __restrict__ in, unsigned int* __restrict__ stats, const int4* __restrict__ ops, int layers,
                int layer, long long hw, const __grid_constant__ RAStatsList list) {
  __shared__ unsigned int hist[768];
  __shared__ unsigned long long lsum;
  const int b = list.img[blockIdx.y];
  const bool histo = __ldg(&ops[(long long)b * layers + layer].x) != kContrast;
  for (int i = threadIdx.x; i < 768; i += blockDim.x) hist[i] = 0;
  if (threadIdx.x == 0) lsum = 0;
  __syncthreads();
  const uint8_t* p = in + (long long)b * hw * 3;
  unsigned long long s = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t r = __ldg(p + i * 3), g = __ldg(p + i * 3 + 1), bl = __ldg(p + i * 3 + 2);
    if (histo) {
      atomicAdd(&hist[r], 1u);
      atomicAdd(&hist[256 + g], 1u);
      atomicAdd(&hist[512 + bl], 1u);
    } else {
      s += ra_luma(r, g, bl);
    }
  }
  if (!histo) atomicAdd(&lsum, s);
  __syncthreads();
  unsigned int* st = stats + (long long)b * kRAStatsWords;
  if (histo) {
    for (int i = threadIdx.x; i < 768; i += blockDim.x)
      if (hist[i]) atomicAdd(st + i, hist[i]);
  } else if (threadIdx.x == 0) {
    atomicAdd(reinterpret_cast<unsigned long long*>(st + 768), lsum);
  }
}

// ImageOps' LUTs for image b (blockDim.x == 256: thread t owns entry t of each channel)
__device__ void ra_build_lut(int op, int iparam, const unsigned int* __restrict__ st, long long hw, uint8_t (*lut)[256]) {
  __shared__ unsigned int cum[3][256];
  __shared__ int lo[3], hi[3], nz[3];
  const int t = threadIdx.x;
  if (op == kInvert || op == kPosterize || op == kSolarize || op == kSolarizeAdd) {
    int v;
    if (op == kInvert) v = 255 - t;
    else if (op == kPosterize) v = t & ~((1 << (8 - iparam)) - 1) & 255;
    else if (op == kSolarize) v = t < iparam ? t : 255 - t;
    else v = t < 128 ? min(255, t + iparam) : t;
    lut[0][t] = lut[1][t] = lut[2][t] = (uint8_t)v;
    return;
  }
  if (t < 3) {
    lo[t] = 256;
    hi[t] = -1;
    nz[t] = 0;
  }
  unsigned int h[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) h[c] = st[c * 256 + t];
  __syncthreads();
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    cum[c][t] = h[c];
    if (h[c]) {
      atomicMin(&lo[c], t);
      atomicMax(&hi[c], t);
      atomicAdd(&nz[c], 1);
    }
  }
  __syncthreads();
  if (op == kAutoContrast) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int v = t;
      if (hi[c] > lo[c]) {   // ImageOps.autocontrast(cutoff=0): int(ix * scale + offset) in float64, clipped
        const double scale = __ddiv_rn(255.0, (double)(hi[c] - lo[c]));
        const double offset = __dmul_rn((double)-lo[c], scale);
        v = (int)__dadd_rn(__dmul_rn((double)t, scale), offset);
        v = v < 0 ? 0 : (v > 255 ? 255 : v);
      }
      lut[c][t] = (uint8_t)v;
    }
    return;
  }
  // Equalize: n // step with n = step // 2 + the count below bin t, step = (pixels - count of the last used bin) // 255
  for (int off = 1; off < 256; off <<= 1) {
    unsigned int v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = t >= off ? cum[c][t - off] : 0u;
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) cum[c][t] += v[c];
    __syncthreads();
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    long long v = t;
    if (nz[c] > 1) {
      const long long step = (hw - (long long)st[c * 256 + hi[c]]) / 255;
      if (step) {
        v = (step / 2 + (long long)(cum[c][t] - h[c])) / step;
        v = v > 255 ? 255 : v;
      }
    }
    lut[c][t] = (uint8_t)v;
  }
}

// Image.blend(degenerate, image, f): float32 deg + f * (img - deg), clipped, truncated (Pillow's Blend.c)
__device__ __forceinline__ uint8_t ra_blend(int deg, int v, float f) {
  const float r = __fadd_rn((float)deg, __fmul_rn(f, (float)(v - deg)));
  return r <= 0.f ? 0 : (r >= 255.f ? 255 : (uint8_t)(int)r);
}

// ImageFilter.SMOOTH at an interior pixel: rows y+1, y, y-1 of (1 1 1 / 1 5 1 / 1 1 1) / 13 in float32, rounded
__device__ __forceinline__ int ra_smooth(const uint8_t* __restrict__ p, int y, int x, int w, int c) {
  const float k1 = 1.0f / 13.0f, k5 = 5.0f / 13.0f;
  float ss = 0.f;
#pragma unroll
  for (int dy = 1; dy >= -1; --dy) {
    const uint8_t* r = p + ((long long)(y + dy) * w + x) * 3 + c;
    const float kc = dy == 0 ? k5 : k1;
    ss = __fadd_rn(ss, __fadd_rn(__fadd_rn(__fmul_rn((float)__ldg(r - 3), k1), __fmul_rn((float)__ldg(r), kc)),
                                 __fmul_rn((float)__ldg(r + 3), k1)));
  }
  return ss <= 0.f ? 0 : (ss >= 255.f ? 255 : (int)__dadd_rn((double)ss, 0.5));
}

// Pillow's bicubic kernel (Geometry.c BICUBIC) in float64
__device__ __forceinline__ double ra_cubic(double v1, double v2, double v3, double v4, double d) {
  const double p2 = __dadd_rn(-v1, v3);
  const double p3 = __dsub_rn(__dadd_rn(__dmul_rn(2.0, __dsub_rn(v1, v2)), v3), v4);
  const double p4 = __dadd_rn(__dsub_rn(__dadd_rn(-v1, v2), v3), v4);
  return __dadd_rn(v2, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

// Image.transform(size, AFFINE, a, resample, fillcolor) at output pixel (x, y): Geometry.c affine_transform + the
// bilinear / bicubic filters, neighbours clamped to the edge
__device__ __forceinline__ void ra_affine(const uint8_t* __restrict__ p, int y, int x, int h, int w, const double* a,
                                          int resample, const int* fill, uint8_t* o) {
  const double xo = x + 0.5, yo = y + 0.5;
  double xin = __dadd_rn(__dadd_rn(__dmul_rn(a[0], xo), __dmul_rn(a[1], yo)), a[2]);
  double yin = __dadd_rn(__dadd_rn(__dmul_rn(a[3], xo), __dmul_rn(a[4], yo)), a[5]);
  if (!(xin >= 0.0 && xin < (double)w && yin >= 0.0 && yin < (double)h)) {
    o[0] = (uint8_t)fill[0], o[1] = (uint8_t)fill[1], o[2] = (uint8_t)fill[2];
    return;
  }
  xin = __dsub_rn(xin, 0.5);
  yin = __dsub_rn(yin, 0.5);
  const int x0 = (int)floor(xin), y0 = (int)floor(yin);
  const double dx = __dsub_rn(xin, (double)x0), dy = __dsub_rn(yin, (double)y0);
  auto at = [&](int yy, int xx, int c) -> int {
    yy = yy < 0 ? 0 : (yy >= h ? h - 1 : yy);
    xx = xx < 0 ? 0 : (xx >= w ? w - 1 : xx);
    return __ldg(p + ((long long)yy * w + xx) * 3 + c);
  };
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double v;
    if (resample == kBilinear) {
      const int p00 = at(y0, x0, c), p01 = at(y0, x0 + 1, c), p10 = at(y0 + 1, x0, c), p11 = at(y0 + 1, x0 + 1, c);
      const double v1 = __dadd_rn((double)p00, __dmul_rn((double)(p01 - p00), dx));
      const double v2 = __dadd_rn((double)p10, __dmul_rn((double)(p11 - p10), dx));
      v = __dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));
    } else {
      double r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        r[j] = ra_cubic(at(y0 + j - 1, x0 - 1, c), at(y0 + j - 1, x0, c), at(y0 + j - 1, x0 + 1, c), at(y0 + j - 1, x0 + 2, c), dx);
      v = ra_cubic(r[0], r[1], r[2], r[3], dy);
    }
    o[c] = v <= 0.0 ? 0 : (v >= 255.0 ? 255 : (uint8_t)(int)v);
  }
}

struct RAFill {
  int rgb[3];
};

// one layer for image blockIdx.y: in -> out (both uint8 [n][h][w][3]); the op is uniform over the block
__global__ void __launch_bounds__(kInThreads)
ra_apply_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const unsigned int* __restrict__ stats,
                const int4* __restrict__ ops, const float* __restrict__ factors, const double* __restrict__ affine,
                int layers, int layer, int h, int w, RAFill fill) {
  __shared__ uint8_t lut[3][256];
  __shared__ int contrast_deg;
  const int b = blockIdx.y;
  const long long rec = (long long)b * layers + layer, hw = (long long)h * w;
  const int4 o = ops[rec];
  const int op = o.x;
  const uint8_t* src = in + (long long)b * hw * 3;
  uint8_t* dst = out + (long long)b * hw * 3;
  const long long first = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (ra_lut(op)) {
    ra_build_lut(op, o.z, stats + (long long)b * kRAStatsWords, hw, lut);
    __syncthreads();
    for (long long i = first; i < hw; i += stride)
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[i * 3 + c] = lut[c][__ldg(src + i * 3 + c)];
  } else if (ra_enhance(op)) {
    const float f = factors[rec];
    if (op == kContrast) {
      if (threadIdx.x == 0) {   // ImageEnhance.Contrast: int(mean(L) + 0.5), the mean in float64
        const unsigned long long s = *reinterpret_cast<const unsigned long long*>(stats + (long long)b * kRAStatsWords + 768);
        contrast_deg = (int)__dadd_rn(__ddiv_rn((double)s, (double)hw), 0.5);
      }
      __syncthreads();
    }
    for (long long i = first; i < hw; i += stride) {
      const int y = (int)(i / w), x = (int)(i - (long long)y * w);
      const int r = __ldg(src + i * 3), g = __ldg(src + i * 3 + 1), bl = __ldg(src + i * 3 + 2);
      const int px[3] = {r, g, bl};
      const bool interior = y > 0 && y < h - 1 && x > 0 && x < w - 1;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        int deg;
        if (op == kBrightness) deg = 0;
        else if (op == kContrast) deg = contrast_deg;
        else if (op == kColor) deg = (int)ra_luma(r, g, bl);
        else deg = interior ? ra_smooth(src, y, x, w, c) : px[c];   // SMOOTH copies the border
        dst[i * 3 + c] = ra_blend(deg, px[c], f);
      }
    }
  } else if (ra_geometric(op)) {
    double a[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) a[k] = affine[rec * 6 + k];
    for (long long i = first; i < hw; i += stride) {
      const int y = (int)(i / w), x = (int)(i - (long long)y * w);
      ra_affine(src, y, x, h, w, a, o.y, fill.rgb, dst + i * 3);
    }
  } else {
    for (long long i = first; i < hw * 3; i += stride) dst[i] = __ldg(src + i);
  }
}

// ---- RandomResizedCrop / Resize + CenterCrop + horizontal flip on the uint8 edge --------------------------------------
// torchvision's PIL path resizes with Image.resize(BILINEAR), i.e. Pillow's ImagingResample for 8-bit images: per axis a
// float64 triangle-filter table normalised and rounded to 22-bit fixed point, a horizontal pass whose results are
// rounded and kept as uint8, then a vertical pass over those with the same rounding.  The host made the crop and the
// draws (classification.common.Uint8RandomResizedCrop / Uint8Resize); per image the kernel reads the source (h, w), the
// full resized size (fh, fw), the window (top, left) of the oh x ow output inside it and the flip flag.  Each output
// pixel depends only on its own taps, so only the window is computed.  A CTA owns a kRsRows x kRsCols tile: it builds
// the tile's coefficients in shared memory, filters the source rows its vertical taps need horizontally in chunks of
// kRsChunk rows and accumulates the vertical pass in registers, so any downscale factor runs in bounded shared memory
// except for the coefficient tables, whose size the host checks.  Every float64 operation is an explicit _rn intrinsic.
constexpr int kRsMaxImages = 512;   // per launch: the geometry travels in the kernel's parameter space
constexpr int kRsRows = 16, kRsCols = 32, kRsChunk = 32;
constexpr int kRsPixelsPerThread = kRsRows * kRsCols / kInThreads;
constexpr int kRsPrecision = 22;    // Pillow's PRECISION_BITS
constexpr int kRsGeomFields = 9;    // src_h, src_w, full_h, full_w, top, left, out_h, out_w, flip

struct RsImage {
  long long off;                    // first byte of the image's [h][w][3] pixels in the packed source
  int h, w, fh, fw, top, left, flip, pad;
};
struct RsBatch {
  RsImage img[kRsMaxImages];
};

__device__ __forceinline__ uint8_t rs_clip8(int v) {
  return v >= (1 << kRsPrecision << 8) ? 255 : (v <= 0 ? 0 : (uint8_t)(v >> kRsPrecision));
}

__device__ __forceinline__ double rs_triangle(double x) {
  if (x < 0.0) x = -x;
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// Resample.c precompute_coeffs + normalize_coeffs_8bpc (bilinear, box = the whole input) for output index xx:
// first tap xmin, n taps, fixed-point weights k[0..n)
__device__ void rs_coeffs(int in_size, int out_size, int xx, int* k, int* xmin_out, int* n_out) {
  const double scale = __ddiv_rn((double)in_size, (double)out_size);
  const double support = scale < 1.0 ? 1.0 : scale;
  const double ss = __ddiv_rn(1.0, support);
  const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
  int xmin = (int)__dadd_rn(__dsub_rn(center, support), 0.5);
  xmin = xmin < 0 ? 0 : xmin;
  int xmax = (int)__dadd_rn(__dadd_rn(center, support), 0.5);
  xmax = xmax > in_size ? in_size : xmax;
  const int n = xmax - xmin;
  double ww = 0.0;
  for (int x = 0; x < n; ++x) ww = __dadd_rn(ww, rs_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < n; ++x) {
    double w = rs_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    const double s = __dmul_rn(w, (double)(1 << kRsPrecision));
    k[x] = (int)(w < 0.0 ? __dadd_rn(-0.5, s) : __dadd_rn(0.5, s));
  }
  *xmin_out = xmin;
  *n_out = n;
}

// one tile of image blockIdx.z; dynamic shared memory: kh [kRsCols][kx], kv [kRsRows][ky] int32, then the uint8 chunk
__global__ void __launch_bounds__(kInThreads)
u8_resample_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ out, int oh, int ow, int kx, int ky,
                   const __grid_constant__ RsBatch g) {
  extern __shared__ int rs_smem[];
  __shared__ int hx0[kRsCols], hn[kRsCols], vy0[kRsRows], vn[kRsRows];
  int* kh = rs_smem;
  int* kv = kh + kRsCols * kx;
  uint8_t* chunk = reinterpret_cast<uint8_t*>(kv + kRsRows * ky);   // [kRsChunk][kRsCols][3] horizontal-pass results
  const RsImage im = g.img[blockIdx.z];
  const int x0 = blockIdx.x * kRsCols, y0 = blockIdx.y * kRsRows;
  const int cols = min(kRsCols, ow - x0), rows = min(kRsRows, oh - y0);
  const int t = threadIdx.x;
  if (t < cols) rs_coeffs(im.w, im.fw, im.left + x0 + t, kh + t * kx, &hx0[t], &hn[t]);
  else if (t >= kRsCols && t < kRsCols + rows) rs_coeffs(im.h, im.fh, im.top + y0 + t - kRsCols, kv + (t - kRsCols) * ky,
                                                         &vy0[t - kRsCols], &vn[t - kRsCols]);
  __syncthreads();
  int ys = vy0[0], ye = 0;
  for (int r = 0; r < rows; ++r) {
    ys = min(ys, vy0[r]);
    ye = max(ye, vy0[r] + vn[r]);
  }
  int acc[kRsPixelsPerThread][3];
#pragma unroll
  for (int i = 0; i < kRsPixelsPerThread; ++i) acc[i][0] = acc[i][1] = acc[i][2] = 1 << (kRsPrecision - 1);
  const uint8_t* s = src + im.off;
  for (int c0 = ys; c0 < ye; c0 += kRsChunk) {
    const int cn = min(kRsChunk, ye - c0);
    for (int i = t; i < cn * kRsCols; i += kInThreads) {
      const int r = i / kRsCols, c = i - r * kRsCols;
      if (c >= cols) continue;
      const uint8_t* p = s + ((long long)(c0 + r) * im.w + hx0[c]) * 3;
      const int* k = kh + c * kx;
      int a0 = 1 << (kRsPrecision - 1), a1 = a0, a2 = a0;
      for (int j = 0; j < hn[c]; ++j) {
        const int kj = k[j];
        a0 += (int)__ldg(p + 3 * j) * kj;
        a1 += (int)__ldg(p + 3 * j + 1) * kj;
        a2 += (int)__ldg(p + 3 * j + 2) * kj;
      }
      uint8_t* q = chunk + (r * kRsCols + c) * 3;
      q[0] = rs_clip8(a0), q[1] = rs_clip8(a1), q[2] = rs_clip8(a2);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kRsPixelsPerThread; ++i) {
      const int px = t + i * kInThreads, r = px / kRsCols, c = px - r * kRsCols;
      if (r >= rows || c >= cols) continue;
      const int lo = max(c0, vy0[r]), hi = min(c0 + cn, vy0[r] + vn[r]);
      const int* k = kv + r * ky;
      for (int y = lo; y < hi; ++y) {
        const uint8_t* q = chunk + ((y - c0) * kRsCols + c) * 3;
        const int kj = k[y - vy0[r]];
        acc[i][0] += (int)q[0] * kj;
        acc[i][1] += (int)q[1] * kj;
        acc[i][2] += (int)q[2] * kj;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < kRsPixelsPerThread; ++i) {
    const int px = t + i * kInThreads, r = px / kRsCols, c = px - r * kRsCols;
    if (r >= rows || c >= cols) continue;
    const int x = im.flip ? ow - 1 - (x0 + c) : x0 + c;
    uint8_t* o = out + (((long long)blockIdx.z * oh + y0 + r) * ow + x) * 3;
    o[0] = rs_clip8(acc[i][0]), o[1] = rs_clip8(acc[i][1]), o[2] = rs_clip8(acc[i][2]);
  }
}

// taps of Pillow's bilinear table for an in_size -> out_size axis: 2 * ceil(support) + 1
int rs_ksize(int in_size, int out_size) {
  const double scale = (double)in_size / (double)out_size;
  return (int)ceil(scale < 1.0 ? 1.0 : scale) * 2 + 1;
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

extern "C" int saicv_u8_rand_augment(void* img, void* scratch, int n, int h, int w, int layers, const int* ops_host,
                                     const float* factors_host, const double* affine_host, const int* ops,
                                     const float* factors, const double* affine, const int* fill3, unsigned int* stats,
                                     void* stream) {
  const char* fn = "saicv_u8_rand_augment";
  if (!img || !scratch || !ops_host || !factors_host || !affine_host || !ops || !factors || !affine || !fill3 || !stats)
    return set_error("%s: null pointer", fn);
  if (img == scratch) return set_error("%s: the scratch buffer must not be the image buffer", fn);
  if (n < 1 || n > kRAMaxImages) return set_error("%s: 1 <= n <= %d (n=%d)", fn, kRAMaxImages, n);
  if (h < 1 || w < 1 || (long long)h * w >= (1ll << 31)) return set_error("%s: image %d x %d is empty or too large", fn, h, w);
  if (layers < 0 || layers > kRAMaxLayers) return set_error("%s: 0 <= layers <= %d (layers=%d)", fn, kRAMaxLayers, layers);
  RAFill fill;
  for (int c = 0; c < 3; ++c) {
    if (fill3[c] < 0 || fill3[c] > 255) return set_error("%s: fill colour component %d is %d, not in [0, 255]", fn, c, fill3[c]);
    fill.rgb[c] = fill3[c];
  }
  for (long long r = 0; r < (long long)n * layers; ++r) {
    const int b = (int)(r / layers), l = (int)(r % layers);
    const int op = ops_host[4 * r], resample = ops_host[4 * r + 1], ip = ops_host[4 * r + 2];
    if (op < kRASkip || op >= kRANumOps) return set_error("%s: image %d layer %d: op %d is not in [-1, %d]", fn, b, l, op, kRANumOps - 1);
    if (ra_geometric(op)) {
      if (resample != kBilinear && resample != kBicubic)
        return set_error("%s: image %d layer %d: resample %d is not BILINEAR (2) or BICUBIC (3)", fn, b, l, resample);
      for (int k = 0; k < 6; ++k)
        if (!isfinite(affine_host[6 * r + k])) return set_error("%s: image %d layer %d: affine coefficient %d is not finite", fn, b, l, k);
    }
    if (ra_enhance(op) && !isfinite(factors_host[r])) return set_error("%s: image %d layer %d: enhance factor is not finite", fn, b, l);
    const int ip_max = op == kPosterize ? 8 : op == kSolarize ? 256 : op == kSolarizeAdd ? 255 : 0;
    if ((op == kPosterize || op == kSolarize || op == kSolarizeAdd) && (ip < 0 || ip > ip_max))
      return set_error("%s: image %d layer %d: iparam %d of op %d is not in [0, %d]", fn, b, l, ip, op, ip_max);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long hw = (long long)h * w;
  const int gx = grid_1d((hw + kRAPixelsPerThread - 1) / kRAPixelsPerThread, kInThreads, 65535);
  uint8_t* buf[2] = {reinterpret_cast<uint8_t*>(img), reinterpret_cast<uint8_t*>(scratch)};
  static thread_local RAStatsList list;
  for (int l = 0; l < layers; ++l) {
    const uint8_t* in = buf[l & 1];
    uint8_t* out = buf[(l + 1) & 1];
    list.count = 0;
    for (int b = 0; b < n; ++b)
      if (ra_needs_stats(ops_host[4 * ((long long)b * layers + l)])) list.img[list.count++] = (unsigned short)b;
    if (list.count) {
      if (cudaMemsetAsync(stats, 0, sizeof(unsigned int) * kRAStatsWords * (size_t)n, st) != cudaSuccess)
        return set_error("%s: cudaMemsetAsync of the statistics failed", fn);
      ra_stats_kernel<<<dim3(gx, list.count), kInThreads, 0, st>>>(in, stats, reinterpret_cast<const int4*>(ops), layers, l, hw, list);
      if (check_launch("ra_stats_kernel")) return 1;
    }
    ra_apply_kernel<<<dim3(gx, n), kInThreads, 0, st>>>(in, out, stats, reinterpret_cast<const int4*>(ops), factors, affine,
                                                         layers, l, h, w, fill);
    if (check_launch("ra_apply_kernel")) return 1;
  }
  if (layers & 1) {   // the last layer wrote the scratch buffer
    if (cudaMemcpyAsync(img, scratch, (size_t)n * hw * 3, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return set_error("%s: copy back from the scratch buffer failed", fn);
  }
  return 0;
}

extern "C" int saicv_u8_resample(const void* src, long long src_len, const long long* offsets, const int* geom, int n,
                                 void* out, int oh, int ow, void* stream) {
  const char* fn = "saicv_u8_resample";
  if (!src || !offsets || !geom || !out) return set_error("%s: null pointer", fn);
  if (n < 1 || oh < 1 || ow < 1 || src_len < 0) return set_error("%s: empty batch or output (n=%d, %d x %d)", fn, n, oh, ow);
  if ((long long)oh * ow >= (1ll << 31)) return set_error("%s: output %d x %d is too large", fn, oh, ow);
  int kx = 1, ky = 1;
  for (int b = 0; b < n; ++b) {
    const int* gm = geom + (long long)b * kRsGeomFields;
    const int h = gm[0], w = gm[1], fh = gm[2], fw = gm[3], top = gm[4], left = gm[5], flip = gm[8];
    const long long off = offsets[b];
    if (h < 1 || w < 1 || fh < 1 || fw < 1)
      return set_error("%s: image %d has an empty source (%d x %d) or resized size (%d x %d)", fn, b, h, w, fh, fw);
    if (off < 0 || off > src_len || (long long)h * w > (src_len - off) / 3)
      return set_error("%s: image %d's %d x %d pixels at offset %lld are past the packed buffer of %lld bytes", fn, b, h, w,
                       off, src_len);
    if (gm[6] != oh || gm[7] != ow)
      return set_error("%s: image %d's window is %d x %d, the output is %d x %d", fn, b, gm[6], gm[7], oh, ow);
    if (top < 0 || left < 0 || (long long)top + oh > fh || (long long)left + ow > fw)
      return set_error("%s: image %d's window (top %d, left %d, %d x %d) leaves the %d x %d resized image", fn, b, top, left, oh,
                       ow, fh, fw);
    if (flip != 0 && flip != 1) return set_error("%s: image %d's flip flag is %d, not 0 or 1", fn, b, flip);
    kx = std::max(kx, rs_ksize(w, fw));
    ky = std::max(ky, rs_ksize(h, fh));
  }
  const size_t smem = sizeof(int) * ((size_t)kRsCols * kx + (size_t)kRsRows * ky) + kRsChunk * kRsCols * 3;
  constexpr size_t kSmemCap = 227 * 1024 - 4 * sizeof(int) * (kRsCols + kRsRows);
  if (smem > kSmemCap)
    return set_error("%s: a downscale by more than %d x %d taps needs %zu bytes of coefficients, over %zu", fn, kx, ky, smem,
                     kSmemCap);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(u8_resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error("%s: %s", fn, cudaGetErrorString(e));
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static thread_local RsBatch batch;
  for (int b0 = 0; b0 < n; b0 += kRsMaxImages) {
    const int count = std::min(kRsMaxImages, n - b0);
    for (int i = 0; i < count; ++i) {
      const int* gm = geom + (long long)(b0 + i) * kRsGeomFields;
      batch.img[i] = RsImage{offsets[b0 + i], gm[0], gm[1], gm[2], gm[3], gm[4], gm[5], gm[8], 0};
    }
    const dim3 grid((ow + kRsCols - 1) / kRsCols, (oh + kRsRows - 1) / kRsRows, count);
    u8_resample_kernel<<<grid, kInThreads, smem, st>>>(reinterpret_cast<const uint8_t*>(src),
                                                       reinterpret_cast<uint8_t*>(out) + (long long)b0 * oh * ow * 3, oh, ow,
                                                       kx, ky, batch);
    if (check_launch("u8_resample_kernel")) return 1;
  }
  return 0;
}
