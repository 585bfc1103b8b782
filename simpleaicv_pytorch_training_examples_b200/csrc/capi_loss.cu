// SAMLoss on full-resolution mask logits (SimpleAICV/interactive_segmentation/losses.py:11-198) as two streaming
// passes.  The reference evaluates sigmoid focal loss, dice loss and the IoU-prediction target with ~25 full-size
// elementwise torch kernels per prompt iteration on [B, M, 1024, 1024] fp32 maps (x 5 iterations per step); here ONE
// pass reduces the six per-(b, m) sums all three terms need, and ONE pass writes the logit gradient:
//   sums[b*M+m] = { S_f = sum focal_weight * bce,  S_pt = sum sigmoid(x) t,  S_p = sum sigmoid(x),  S_t = sum t,
//                   I = #(x > thr & t > thr),  U = #(x > thr | t > thr) }
//   focal[b,m] = S_f / (N B)   dice[b,m] = (1 - (2 S_pt + 1) / (S_p + S_t + 1)) / B   gt_iou = clamp(I / max(U, 1e-6), 0, 1)
//   dL/dx = cf[b,m] * d(focal_weight * bce)/dx + sigmoid'(x) * (c1[b,m] * t + c2[b,m])
// HBM-bound: 8 B/pixel forward (fp32 logits + fp32 target; the target plane is shared by the M masks of an image and
// mostly L2-resident), 12 B/pixel backward.  Reductions are per-block partials folded in a fixed order (bit-reproducible).
#include <climits>

#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"

namespace saicv {
namespace {

constexpr int kLossThreads = 256;
constexpr int kMaxBlocksPerPlane = 64;

__device__ __forceinline__ float4 load4(const void* p, long long i4, bool bf16) {
  if (!bf16) return __ldg(reinterpret_cast<const float4*>(p) + i4);
  const uint2 w = __ldg(reinterpret_cast<const uint2*>(p) + i4);
  return make_float4(__uint_as_float(w.x << 16), __uint_as_float(w.x & 0xffff0000u), __uint_as_float(w.y << 16),
                     __uint_as_float(w.y & 0xffff0000u));
}

struct PixelTerms {
  float focal, sig;
};
// focal_weight * bce and sigmoid of one pixel (losses.py:126-141)
__device__ __forceinline__ PixelTerms pixel_terms(float x, float t, float alpha, float gamma) {
  const float e = __expf(-fabsf(x));
  const float inv = __fdividef(1.f, 1.f + e);
  const float sig = x >= 0.f ? inv : e * inv;
  const float bce = fmaxf(x, 0.f) - x * t + log1pf(e);
  const float pt = sig * t + (1.f - sig) * (1.f - t);
  const float af = alpha * t + (1.f - alpha) * (1.f - t);
  const float om = 1.f - pt;
  const float w = gamma == 2.f ? om * om : powf(om, gamma);
  return {af * w * bce, sig};
}

__global__ void __launch_bounds__(kLossThreads)
sam_loss_sums_kernel(const void* __restrict__ logits, int logits_bf16, const float* __restrict__ targets, float* __restrict__ partials,
                     int M, long long n4, float alpha, float gamma, float thr) {
  const int plane = blockIdx.y;                    // b * M + m
  const int b = plane / M;
  const size_t esz = logits_bf16 ? 2 : 4;
  const char* lp = reinterpret_cast<const char*>(logits) + (size_t)plane * n4 * 4 * esz;
  const float4* tp = reinterpret_cast<const float4*>(targets) + (long long)b * n4;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 x = load4(lp, i, logits_bf16 != 0);
    const float4 t = __ldg(tp + i);
    const float xs[4] = {x.x, x.y, x.z, x.w}, ts[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const PixelTerms pt = pixel_terms(xs[k], ts[k], alpha, gamma);
      s[0] += pt.focal;
      s[1] += pt.sig * ts[k];
      s[2] += pt.sig;
      s[3] += ts[k];
      const bool px = xs[k] > thr, tx = ts[k] > thr;
      s[4] += (px && tx) ? 1.f : 0.f;
      s[5] += (px || tx) ? 1.f : 0.f;
    }
  }
  __shared__ float red[kLossThreads / 32][6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float v = s[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kLossThreads / 32; ++w) v += red[w][threadIdx.x];
    partials[((long long)plane * gridDim.x + blockIdx.x) * 6 + threadIdx.x] = v;
  }
}

__global__ void sam_loss_fold_kernel(const float* __restrict__ partials, float* __restrict__ sums, int planes, int nblk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // plane * 6 + k
  if (i >= planes * 6) return;
  const int plane = i / 6, k = i % 6;
  float v = 0.f;
  for (int b = 0; b < nblk; ++b) v += partials[((long long)plane * nblk + b) * 6 + k];
  sums[i] = v;
}

// dlogits = cf * d(focal_weight * bce)/dx + sigmoid'(x) * (c1 * t + c2), coefficients per plane in coef[plane][3]
__global__ void __launch_bounds__(kLossThreads)
sam_loss_bwd_kernel(const void* __restrict__ logits, int logits_bf16, const float* __restrict__ targets, const float* __restrict__ coef,
                    void* __restrict__ dlogits, int dl_bf16, int M, long long n4, float alpha, float gamma) {
  const int plane = blockIdx.y;
  const int b = plane / M;
  const size_t esz = logits_bf16 ? 2 : 4;
  const char* lp = reinterpret_cast<const char*>(logits) + (size_t)plane * n4 * 4 * esz;
  const float4* tp = reinterpret_cast<const float4*>(targets) + (long long)b * n4;
  const float cf = coef[plane * 3], c1 = coef[plane * 3 + 1], c2 = coef[plane * 3 + 2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 x = load4(lp, i, logits_bf16 != 0);
    const float4 t = __ldg(tp + i);
    const float xs[4] = {x.x, x.y, x.z, x.w}, ts[4] = {t.x, t.y, t.z, t.w};
    float g[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xv = xs[k], tv = ts[k];
      const float e = __expf(-fabsf(xv));
      const float inv = __fdividef(1.f, 1.f + e);
      const float sig = xv >= 0.f ? inv : e * inv;
      const float ds = sig * (1.f - sig);
      const float bce = fmaxf(xv, 0.f) - xv * tv + log1pf(e);
      const float pt = sig * tv + (1.f - sig) * (1.f - tv);
      const float af = alpha * tv + (1.f - alpha) * (1.f - tv);
      const float om = 1.f - pt;
      float w, dw;                                  // (1 - pt)^gamma and its derivative w.r.t. pt, negated below
      if (gamma == 2.f) {
        w = om * om;
        dw = 2.f * om;
      } else {
        w = powf(om, gamma);
        dw = om > 0.f ? gamma * powf(om, gamma - 1.f) : 0.f;
      }
      const float dpt = ds * (2.f * tv - 1.f);
      const float dfocal = af * (-dw * dpt * bce + w * (sig - tv));
      g[k] = cf * dfocal + ds * (c1 * tv + c2);
    }
    if (dl_bf16) {
      __nv_bfloat162 a = __floats2bfloat162_rn(g[0], g[1]), c = __floats2bfloat162_rn(g[2], g[3]);
      reinterpret_cast<uint2*>(reinterpret_cast<char*>(dlogits) + (size_t)plane * n4 * 8)[i] =
          make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&c));
    } else {
      reinterpret_cast<float4*>(reinterpret_cast<char*>(dlogits) + (size_t)plane * n4 * 16)[i] = make_float4(g[0], g[1], g[2], g[3]);
    }
  }
}

int blocks_per_plane(long long n4) {
  long long b = (n4 + kLossThreads * 4 - 1) / (kLossThreads * 4);
  if (b < 1) b = 1;
  if (b > kMaxBlocksPerPlane) b = kMaxBlocksPerPlane;
  return (int)b;
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_sam_loss_partial_floats(int b, int m, long long n) { return b * m * blocks_per_plane(n / 4) * 6; }

int saicv_sam_loss_sums(const void* logits, int logits_bf16, const float* targets, float* partials, float* sums, int b, int m,
                        long long n, float alpha, float gamma, float mask_threshold, void* stream) {
  if (n % 4 || n <= 0) return set_error("saicv_sam_loss_sums: the plane size must be a positive multiple of 4 (got %lld)", n);
  const int nblk = blocks_per_plane(n / 4);
  sam_loss_sums_kernel<<<dim3(nblk, b * m), kLossThreads, 0, ST>>>(logits, logits_bf16, targets, partials, m, n / 4, alpha, gamma,
                                                                    mask_threshold);
  if (int e = check_launch("sam_loss_sums_kernel")) return e;
  sam_loss_fold_kernel<<<(b * m * 6 + 127) / 128, 128, 0, ST>>>(partials, sums, b * m, nblk);
  return check_launch("sam_loss_fold_kernel");
}

int saicv_sam_loss_bwd(const void* logits, int logits_bf16, const float* targets, const float* coef, void* dlogits, int dl_bf16, int b,
                       int m, long long n, float alpha, float gamma, void* stream) {
  if (n % 4 || n <= 0) return set_error("saicv_sam_loss_bwd: the plane size must be a positive multiple of 4 (got %lld)", n);
  const int nblk = blocks_per_plane(n / 4);
  sam_loss_bwd_kernel<<<dim3(nblk, b * m), kLossThreads, 0, ST>>>(logits, logits_bf16, targets, coef, dlogits, dl_bf16, m, n / 4, alpha,
                                                                   gamma);
  return check_launch("sam_loss_bwd_kernel");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// SemanticSoftmaxLoss of the ImageNet-21K semantic-tree training (SimpleAICV/classification/losses.py:94-140) and the
// accuracy of SemanticSoftmaxMeter (classification/common.py:712-757) on the full [B, N] logits.  Level l owns the sorted
// columns level_cols[level_off[l] .. level_off[l+1]) (n_l of them); a column belongs to at most one level.  The reference
// gathers outputs[:, index_l] and runs ~14 torch kernels per level; here one CTA per row walks every level's columns once:
//   lse[b,l]  = log sum_{c in l} exp(x_c)
//   loss_bl   = v_bl * (lse - (1-s) x_{y_bl} - (s/n_l) sum_{c in l} x_c)           (v_bl = y_bl >= 0)
//   loss      = sum_l factor_l * (sum_b loss_bl) / B                               (level order, batch folded in order)
//   dL/dx_c   = g factor_l / B * v_bl * (exp(x_c - lse_bl) - s/n_l - (1-s) [c == y_bl])   (0 outside every level)
// Reads each logit once per pass (~42 KB per row at N = 10 450); no float atomics, so the loss is bit-reproducible.
namespace saicv {
namespace {

constexpr int kSemThreads = 256;
constexpr int kSemWarps = kSemThreads / 32;
constexpr int kSemMaxLevels = 16;

__device__ __forceinline__ float sem_load(const void* row, int c, bool bf16) {
  if (bf16) return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(row) + c) << 16);
  return __ldg(reinterpret_cast<const float*>(row) + c);
}

// (max, sum of exp(x - max)) of two partial log-sum-exps
__device__ __forceinline__ void lse_merge(float& m, float& s, float mo, float so) {
  const float mx = fmaxf(m, mo);
  if (mx == -INFINITY) return;
  s = s * expf(m - mx) + so * expf(mo - mx);
  m = mx;
}

__global__ void __launch_bounds__(kSemThreads)
semantic_softmax_fwd_kernel(const void* __restrict__ logits, int logits_bf16, const long long* __restrict__ labels,
                            const int* __restrict__ level_cols, const int* __restrict__ level_off, float* __restrict__ lse,
                            float* __restrict__ terms, int n, int levels, float smoothing) {
  const int row = blockIdx.x;
  const bool bf16 = logits_bf16 != 0;
  const char* xrow = reinterpret_cast<const char*>(logits) + (size_t)row * n * (bf16 ? 2 : 4);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float red[3][kSemWarps];
  for (int lv = 0; lv < levels; ++lv) {
    const int c0 = level_off[lv], c1 = level_off[lv + 1];
    float m = -INFINITY, s = 0.f, sx = 0.f;
    for (int i = c0 + threadIdx.x; i < c1; i += kSemThreads) {
      const float x = sem_load(xrow, __ldg(level_cols + i), bf16);
      sx += x;
      if (x > m) {
        s = s * expf(m - x) + 1.f;
        m = x;
      } else {
        s += expf(x - m);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, m, o), so = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, mo, so);
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
    }
    if (lane == 0) {
      red[0][warp] = m;
      red[1][warp] = s;
      red[2][warp] = sx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float M = red[0][0], S = red[1][0], SX = red[2][0];
      for (int w = 1; w < kSemWarps; ++w) {
        lse_merge(M, S, red[0][w], red[1][w]);
        SX += red[2][w];
      }
      const int nl = c1 - c0;
      const long long y = labels[(long long)row * levels + lv];
      const int yi = y < 0 ? 0 : (y >= nl ? nl - 1 : (int)y);     // the reference scores label 0 on invalid rows
      const float l = M + logf(S);
      const float xy = sem_load(xrow, level_cols[c0 + yi], bf16);
      const float t = l - (1.f - smoothing) * xy - smoothing / (float)nl * SX;
      lse[(long long)row * levels + lv] = l;
      terms[(long long)row * levels + lv] = (y >= 0 ? 1.f : 0.f) * t;   // 0 * NaN stays NaN, as in the reference
    }
    __syncthreads();
  }
}

// loss = sum_l factor_l * mean_b terms[b, l]: warp w folds levels w, w + 8, ...; thread 0 sums the levels in order
__global__ void __launch_bounds__(kSemThreads)
semantic_softmax_fold_kernel(const float* __restrict__ terms, const float* __restrict__ factors, float* __restrict__ loss, int b,
                             int levels) {
  __shared__ float level_sum[kSemMaxLevels];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int lv = warp; lv < levels; lv += kSemWarps) {
    float v = 0.f;
    for (int r = lane; r < b; r += 32) v += terms[(long long)r * levels + lv];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) level_sum[lv] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float total = 0.f;
    for (int lv = 0; lv < levels; ++lv) total += level_sum[lv] / (float)b * factors[lv];
    *loss = total;
  }
}

__global__ void __launch_bounds__(kSemThreads)
semantic_softmax_bwd_kernel(const void* __restrict__ logits, int logits_bf16, const long long* __restrict__ labels,
                            const int* __restrict__ col_level, const int* __restrict__ level_cols, const int* __restrict__ level_off,
                            const float* __restrict__ factors, const float* __restrict__ lse, const float* __restrict__ grad,
                            float* __restrict__ dlogits, int b, int n, int levels, float smoothing) {
  const int row = blockIdx.y;
  const bool bf16 = logits_bf16 != 0;
  const char* xrow = reinterpret_cast<const char*>(logits) + (size_t)row * n * (bf16 ? 2 : 4);
  __shared__ float s_lse[kSemMaxLevels], s_coef[kSemMaxLevels], s_sn[kSemMaxLevels];
  __shared__ int s_ycol[kSemMaxLevels];
  if (threadIdx.x < levels) {
    const int lv = threadIdx.x;
    const int c0 = level_off[lv], nl = level_off[lv + 1] - c0;
    const long long y = labels[(long long)row * levels + lv];
    s_lse[lv] = lse[(long long)row * levels + lv];
    s_coef[lv] = y >= 0 ? *grad * factors[lv] / (float)b : 0.f;
    s_sn[lv] = smoothing / (float)nl;
    s_ycol[lv] = (y >= 0 && y < nl) ? level_cols[c0 + (int)y] : -1;
  }
  __syncthreads();
  float* drow = dlogits + (long long)row * n;
  for (int c = blockIdx.x * kSemThreads + threadIdx.x; c < n; c += gridDim.x * kSemThreads) {
    const int lv = __ldg(col_level + c);
    float g = 0.f;
    if (lv >= 0 && s_coef[lv] != 0.f) {
      const float p = expf(sem_load(xrow, c, bf16) - s_lse[lv]);
      g = s_coef[lv] * (p - s_sn[lv] - (c == s_ycol[lv] ? 1.f - smoothing : 0.f));
    }
    drow[c] = g;
  }
}

// counts[l] = {#rows whose first argmax over level l's columns equals the label, #rows with a label >= 0}; NaN counts as
// the maximum and the first of equal maxima wins (torch.argmax)
__device__ __forceinline__ bool argmax_better(float v1, int i1, float v2, int i2) {
  const bool n1 = isnan(v1), n2 = isnan(v2);
  if (n1 != n2) return n1;
  if (!n1 && v1 != v2) return v1 > v2;
  return i1 < i2;
}

__global__ void __launch_bounds__(kSemThreads)
semantic_accuracy_kernel(const void* __restrict__ logits, int logits_bf16, const long long* __restrict__ labels,
                         const int* __restrict__ level_cols, const int* __restrict__ level_off, int* __restrict__ counts, int n,
                         int levels) {
  const int row = blockIdx.x;
  const bool bf16 = logits_bf16 != 0;
  const char* xrow = reinterpret_cast<const char*>(logits) + (size_t)row * n * (bf16 ? 2 : 4);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float rv[kSemWarps];
  __shared__ int ri[kSemWarps];
  for (int lv = 0; lv < levels; ++lv) {
    const int c0 = level_off[lv], c1 = level_off[lv + 1];
    float v = -INFINITY;
    int idx = INT_MAX;
    for (int i = c0 + threadIdx.x; i < c1; i += kSemThreads) {
      const float x = sem_load(xrow, __ldg(level_cols + i), bf16);
      if (argmax_better(x, i - c0, v, idx)) {
        v = x;
        idx = i - c0;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float vo = __shfl_xor_sync(0xffffffffu, v, o);
      const int io = __shfl_xor_sync(0xffffffffu, idx, o);
      if (argmax_better(vo, io, v, idx)) {
        v = vo;
        idx = io;
      }
    }
    if (lane == 0) {
      rv[warp] = v;
      ri[warp] = idx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kSemWarps; ++w)
        if (argmax_better(rv[w], ri[w], v, idx)) {
          v = rv[w];
          idx = ri[w];
        }
      const long long y = labels[(long long)row * levels + lv];
      if (y >= 0) {
        atomicAdd(counts + 2 * lv + 1, 1);
        if ((long long)idx == y) atomicAdd(counts + 2 * lv, 1);
      }
    }
    __syncthreads();
  }
}

int semantic_check(const char* what, int b, int n, int levels) {
  if (b <= 0 || n <= 0) return set_error("%s: empty logits [%d, %d]", what, b, n);
  if (levels <= 0 || levels > kSemMaxLevels) return set_error("%s: %d levels (1..%d supported)", what, levels, kSemMaxLevels);
  return 0;
}

}  // namespace
}  // namespace saicv

extern "C" {

int saicv_semantic_softmax_fwd(const void* logits, int logits_bf16, const long long* labels, const int* level_cols,
                               const int* level_off, const float* factors, float* lse, float* terms, float* loss, int b, int n,
                               int levels, float smoothing, void* stream) {
  if (int e = semantic_check("saicv_semantic_softmax_fwd", b, n, levels)) return e;
  semantic_softmax_fwd_kernel<<<b, kSemThreads, 0, ST>>>(logits, logits_bf16, labels, level_cols, level_off, lse, terms, n, levels,
                                                         smoothing);
  if (int e = check_launch("semantic_softmax_fwd_kernel")) return e;
  semantic_softmax_fold_kernel<<<1, kSemThreads, 0, ST>>>(terms, factors, loss, b, levels);
  return check_launch("semantic_softmax_fold_kernel");
}

int saicv_semantic_softmax_bwd(const void* logits, int logits_bf16, const long long* labels, const int* col_level,
                               const int* level_cols, const int* level_off, const float* factors, const float* lse,
                               const float* grad, float* dlogits, int b, int n, int levels, float smoothing, void* stream) {
  if (int e = semantic_check("saicv_semantic_softmax_bwd", b, n, levels)) return e;
  const int col_blocks = (n + kSemThreads * 4 - 1) / (kSemThreads * 4);
  semantic_softmax_bwd_kernel<<<dim3(col_blocks, b), kSemThreads, 0, ST>>>(logits, logits_bf16, labels, col_level, level_cols,
                                                                            level_off, factors, lse, grad, dlogits, b, n, levels,
                                                                            smoothing);
  return check_launch("semantic_softmax_bwd_kernel");
}

int saicv_semantic_accuracy(const void* logits, int logits_bf16, const long long* labels, const int* level_cols,
                            const int* level_off, int* counts, int b, int n, int levels, void* stream) {
  if (int e = semantic_check("saicv_semantic_accuracy", b, n, levels)) return e;
  if (cudaMemsetAsync(counts, 0, sizeof(int) * 2 * levels, ST) != cudaSuccess)
    return set_error("saicv_semantic_accuracy: clearing the counts failed");
  semantic_accuracy_kernel<<<b, kSemThreads, 0, ST>>>(logits, logits_bf16, labels, level_cols, level_off, counts, n, levels);
  return check_launch("semantic_accuracy_kernel");
}

}  // extern "C"
