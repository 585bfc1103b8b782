// HBM-bound kernels of the conv-net hot path: BatchNorm (training) statistics / apply /
// backward, ReLU + residual fusion, pooling, layout and weight preparation.  All activations
// are NHWC bf16 viewed as [rows][C]; every thread moves 16-byte vectors (8 x bf16), channel is the
// fastest dimension so warps read/write fully coalesced 512 B segments.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/saicv_b200.h"
#include "host_util.h"
#include "vec8.cuh"

namespace saicv {

static thread_local char g_err[512] = "";
int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s: %s", what, cudaGetErrorString(e));
  count_launch(1);
  return 0;
}
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }
const char* last_error() { return g_err; }
long long launch_count();

namespace {

constexpr int kThreads = 256;

// act: 0 none, 1 ReLU, 2 LeakyReLU(0.1), 3 SiLU (darknet.py:16-31 ActivationBlock)
__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == 3) return v * __fdividef(1.f, 1.f + __expf(-v));
  return act == 1 ? fmaxf(v, 0.f) : (act == 2 ? (v > 0.f ? v : 0.1f * v) : v);
}
__device__ __forceinline__ float act_grad(float out, int act) {
  // ReLU / LeakyReLU: derivative expressed through the activated output OR the pre-activation (same
  // sign).  SiLU: `out` must be the pre-activation z (mask-recompute path only, enforced by the C ABI):
  // silu'(z) = s(z) * (1 + z * (1 - s(z))).
  if (act == 3) {
    const float sg = __fdividef(1.f, 1.f + __expf(-out));
    return sg * (1.f + out * (1.f - sg));
  }
  return act == 1 ? (out > 0.f ? 1.f : 0.f) : (act == 2 ? (out > 0.f ? 1.f : 0.1f) : 1.f);
}

int grid_for(long long work_items, int per_block = kThreads, int max_blocks = 132 * 16) {
  long long b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}
int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// ----------------------------------------------------------------------------- slab kernels
// All BatchNorm kernels share one thread layout: a block owns a slab of rows; thread (tx, ty)
// always handles the same 8 channels (vector tx of every row) and walks rows ty, ty+ty_count, ...
// so per-channel coefficients live in registers for the whole kernel, and UNROLL independent
// 16-byte loads are in flight per tensor per thread.
constexpr int UNROLL = 4;

struct SlabGeom {
  int vpr, tx_count, ty_count;
  long long rows_per_block;
  int ldv;  // row stride in 16-byte vectors (== vpr unless a column chunk of a wider matrix is reduced)
};

// Tree-folds the ty rows of red[][] that share a channel vector and writes this block's partial row(s):
// prow[c] = sum s0, and prow[C + c] = sum s1 unless ONLY_S0.  Every BatchNorm reduction folds through here so that the
// single- and two-BatchNorm backward reductions produce bit-identical partial rows.
template <bool ONLY_S0>
__device__ __forceinline__ void fold_slab(float (*red)[17], const float (&s0)[8], const float (&s1)[8], int tx, int ty,
                                          const SlabGeom& gm, float* __restrict__ prow, int C) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red[threadIdx.x][i] = s0[i];
    red[threadIdx.x][8 + i] = s1[i];
  }
  __syncthreads();
  // tree-fold the ty rows that share a channel vector
  for (int half = gm.ty_count >> 1; half > 0; half >>= 1) {
    if (ty < half) {
#pragma unroll
      for (int i = 0; i < 16; ++i) red[threadIdx.x][i] += red[threadIdx.x + half * gm.tx_count][i];
    }
    __syncthreads();
  }
  // deterministic: one partial row per block, folded later by fold_partials / bn_finalize
  if (ty == 0 && tx < gm.vpr) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      prow[tx * 8 + i] = red[threadIdx.x][i];
      if (!ONLY_S0) prow[C + tx * 8 + i] = red[threadIdx.x][8 + i];
    }
  }
}

// ReLU mask of 8 channels packed as one byte (bit i: channel 8*tx + i, set where the activated output is > 0).  A row of
// C channels is C/8 bytes, so the bytes of channels 32w .. 32w+31 form the little-endian uint32 word w of the
// [rows][C/32] mask that bn_apply writes and the data-gradient GEMM epilogue reads (EPI_MASK_BITS).
__device__ __forceinline__ float mask_bit(uint32_t m, int i) { return ((m >> i) & 1u) ? 1.f : 0.f; }

// MODE 0: sum x, sum x^2 (BN forward statistics)
// MODE 1: g = dout*act'(.); sum g, sum g*xhat (BN backward reductions)
// MODE 2: sum x only (bias gradients)
// Activation mask source for MODE 1: `b` (activated output) when non-null, else the packed ReLU mask `bits` when
// non-null, else recomputed from y with scale/shift `ss` (out = act(y*scale+shift) has the sign of y*scale+shift).
template <int MODE, int UNR>
__global__ void __launch_bounds__(kThreads, 2)
colreduce_kernel(const void* __restrict__ a, const void* __restrict__ b, const uint8_t* __restrict__ bits,
                 const void* __restrict__ y, const float* __restrict__ saved, const float* __restrict__ ss,
                 float* __restrict__ out, long long rows, int C, SlabGeom gm, int act) {
  __shared__ float red[kThreads][17];
  const int vpr = gm.vpr;
  const int tx = threadIdx.x % gm.tx_count;
  const int ty = threadIdx.x / gm.tx_count;
  const int ty_count = gm.ty_count;
  float s0[8], s1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s0[i] = s1[i] = 0.f;
  const long long r0 = (long long)blockIdx.x * gm.rows_per_block;
  long long r1 = r0 + gm.rows_per_block;
  if (r1 > rows) r1 = rows;
  if (tx < vpr) {
    float mean[8], rstd[8], sc[8], sh[8];
    const bool use_bits = (MODE == 1) && act != 0 && b == nullptr && bits != nullptr;
    const bool recompute_mask = (MODE == 1) && act != 0 && b == nullptr && bits == nullptr;
    if (MODE == 1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mean[i] = saved[tx * 8 + i];
        rstd[i] = saved[C + tx * 8 + i];
        sc[i] = recompute_mask ? ss[tx * 8 + i] : 0.f;
        sh[i] = recompute_mask ? ss[C + tx * 8 + i] : 0.f;
      }
    }
    for (long long r = r0 + ty; r < r1; r += (long long)ty_count * UNR) {
      V8 va[UNR], vb[UNR], vy[UNR];
      uint32_t mb[UNR];
      bool ok[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const long long rr = r + (long long)u * ty_count;
        ok[u] = rr < r1;
        if (ok[u]) {
          const long long vi = rr * gm.ldv + tx;
          va[u] = ldg8(a, vi);
          if (MODE == 1) {
            vy[u] = ldg8(y, vi);
            if (use_bits) mb[u] = __ldg(bits + vi);
            else if (act != 0 && !recompute_mask) vb[u] = ldg8(b, vi);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        if (!ok[u]) continue;
        float fa[8];
        unpack8(va[u], fa);
        if (MODE == 0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            s0[i] += fa[i];
            s1[i] += fa[i] * fa[i];
          }
        } else if (MODE == 2) {
#pragma unroll
          for (int i = 0; i < 8; ++i) s0[i] += fa[i];
        } else {
          float fy[8];
          unpack8(vy[u], fy);
          if (act != 0) {
            if (recompute_mask) {
#pragma unroll
              for (int i = 0; i < 8; ++i) fa[i] *= act_grad(fy[i] * sc[i] + sh[i], act);
            } else if (use_bits) {
#pragma unroll
              for (int i = 0; i < 8; ++i) fa[i] *= mask_bit(mb[u], i);
            } else {
              float fo[8];
              unpack8(vb[u], fo);
#pragma unroll
              for (int i = 0; i < 8; ++i) fa[i] *= act_grad(fo[i], act);
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            s0[i] += fa[i];
            s1[i] += fa[i] * (fy[i] - mean[i]) * rstd[i];
          }
        }
      }
    }
  }
  fold_slab<MODE == 2>(red, s0, s1, tx, ty, gm, out + (long long)blockIdx.x * (MODE == 2 ? C : 2 * C), C);
}

// Backward reductions of two BatchNorms that share the gradient g and the row geometry (bn3 and the downsample BN of a
// residual block: both normalise what is summed into the block output).  g is read once; each BatchNorm gets exactly
// the partial rows colreduce_kernel<1> would write for it: BatchNorm A in out[blk][0 .. 2C), B in out[blk][2C .. 4C).
// `bits`: ReLU mask applied to g (null: g arrives masked).
__global__ void __launch_bounds__(kThreads, 2)
colreduce2_kernel(const void* __restrict__ g, const uint8_t* __restrict__ bits, const void* __restrict__ ya,
                  const void* __restrict__ yb, const float* __restrict__ saved_a, const float* __restrict__ saved_b,
                  float* __restrict__ out, long long rows, int C, SlabGeom gm) {
  // Two rows per pass instead of colreduce_kernel<1>'s four keeps the four accumulator sets in registers.  A thread still
  // sums rows ty, ty + ty_count, ... in ascending order: the order depends on the slab geometry only.
  constexpr int UNR = 2;
  __shared__ float red[kThreads][17];
  const int vpr = gm.vpr;
  const int tx = threadIdx.x % gm.tx_count;
  const int ty = threadIdx.x / gm.tx_count;
  const int ty_count = gm.ty_count;
  float sa0[8], sa1[8], sb0[8], sb1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sa0[i] = sa1[i] = sb0[i] = sb1[i] = 0.f;
  const long long r0 = (long long)blockIdx.x * gm.rows_per_block;
  long long r1 = r0 + gm.rows_per_block;
  if (r1 > rows) r1 = rows;
  if (tx < vpr) {
    float ma[8], ra[8], mbn[8], rb[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      ma[i] = saved_a[tx * 8 + i];
      ra[i] = saved_a[C + tx * 8 + i];
      mbn[i] = saved_b[tx * 8 + i];
      rb[i] = saved_b[C + tx * 8 + i];
    }
    for (long long r = r0 + ty; r < r1; r += (long long)ty_count * UNR) {
      V8 vg[UNR], va[UNR], vb[UNR];
      uint32_t mk[UNR];
      bool ok[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const long long rr = r + (long long)u * ty_count;
        ok[u] = rr < r1;
        if (ok[u]) {
          const long long vi = rr * vpr + tx;
          vg[u] = ldg8(g, vi);
          va[u] = ldg8(ya, vi);
          vb[u] = ldg8(yb, vi);
          if (bits) mk[u] = __ldg(bits + vi);
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        if (!ok[u]) continue;
        float fg[8], fa[8], fb[8];
        unpack8(vg[u], fg);
        unpack8(va[u], fa);
        unpack8(vb[u], fb);
        if (bits) {
#pragma unroll
          for (int i = 0; i < 8; ++i) fg[i] *= mask_bit(mk[u], i);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          sa0[i] += fg[i];
          sa1[i] += fg[i] * (fa[i] - ma[i]) * ra[i];
          sb0[i] += fg[i];
          sb1[i] += fg[i] * (fb[i] - mbn[i]) * rb[i];
        }
      }
    }
  }
  float* const prow = out + (long long)blockIdx.x * 4 * C;
  fold_slab<false>(red, sa0, sa1, tx, ty, gm, prow, C);
  fold_slab<false>(red, sb0, sb1, tx, ty, gm, prow + 2 * C, C);
}

// out[j] (+)= sum_b partial[b][j]: 8 columns x 32 row groups per block (the <= 264 partial rows are
// spread over 32 threads per column so the fold is a handful of loads deep)
__global__ void fold_partials_kernel(const float* __restrict__ partial, float* __restrict__ out, int nblk, int ncols,
                                     int accumulate) {
  __shared__ float sm[32][9];
  const int cl = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int col = blockIdx.x * 8 + cl;
  float s = 0.f;
  if (col < ncols)
    for (int b = grp; b < nblk; b += 32) s += partial[(long long)b * ncols + col];
  sm[grp][cl] = s;
  __syncthreads();
  if (grp == 0 && col < ncols) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < 32; ++g) t += sm[g][cl];
    out[col] = accumulate ? out[col] + t : t;
  }
}

constexpr int kMaxPartials = SAICV_BN_PARTIAL_ROWS;  // 2 blocks per SM

bool slab_geom(long long rows, int C, int unroll, SlabGeom* g, int* blocks, int max_blocks = 132 * 8) {
  const int min_rows_per_thread = unroll;
  if (C % 8 || C > 2048) {
    set_error("BatchNorm / column kernels need C %% 8 == 0 and C <= 2048 (C=%d)", C);
    return false;
  }
  g->vpr = C / 8;
  g->ldv = C / 8;
  g->tx_count = next_pow2(g->vpr) > kThreads ? kThreads : next_pow2(g->vpr);
  g->ty_count = kThreads / g->tx_count;
  long long b = (rows + (long long)g->ty_count * min_rows_per_thread - 1) / ((long long)g->ty_count * min_rows_per_thread);
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  g->rows_per_block = (rows + b - 1) / b;
  // keep slabs a multiple of ty_count*UNROLL rows so only the last block has a ragged tail
  const long long q = (long long)g->ty_count * unroll;
  g->rows_per_block = (g->rows_per_block + q - 1) / q * q;
  *blocks = (int)((rows + g->rows_per_block - 1) / g->rows_per_block);
  return true;
}

// Writes `*nblk` partial rows into `partials` ([kMaxPartials][2C] or [..][C] for MODE 2).
template <int MODE>
int launch_colreduce(const void* a, const void* b, const void* y, const float* saved, const float* ss,
                     float* partials, long long rows, int C, int act, int* nblk, cudaStream_t st,
                     const uint32_t* bits = nullptr) {
  SlabGeom g;
  constexpr int UNR = MODE == 1 ? 4 : 8;  // independent 16-byte loads in flight per tensor per thread
  if (!slab_geom(rows, C, UNR, &g, nblk, kMaxPartials)) return 1;
  colreduce_kernel<MODE, UNR><<<*nblk, kThreads, 0, st>>>(a, b, reinterpret_cast<const uint8_t*>(bits), y, saved, ss,
                                                         partials, rows, C, g, act);
  return check_launch("colreduce_kernel");
}
int partial_rows(long long rows, int C) {  // must mirror launch_colreduce<0>
  SlabGeom g;
  int n = 0;
  slab_geom(rows, C, 8, &g, &n, kMaxPartials);
  return n;
}
int fold(const float* partials, float* out, int nblk, int ncols, int accumulate, cudaStream_t st) {
  fold_partials_kernel<<<(ncols + 7) / 8, 256, 0, st>>>(partials, out, nblk, ncols, accumulate);
  return check_launch("fold_partials_kernel");
}

// fp32 column sums (fc bias gradient from fp32 dlogits): small, one thread per column
__global__ void colsum_f32_kernel(const float* __restrict__ x, float* __restrict__ out, long long rows,
                                  int C, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (long long r = 0; r < rows; ++r) s += x[r * C + c];
  out[c] = accumulate ? out[c] + s : s;
}

// ----------------------------------------------------------------------------- BN finalize
// Folds the per-block partial sums (deterministic order) and finalises 8 channels per block.
__global__ void bn_finalize_kernel(const float* __restrict__ partials, int nblk, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* __restrict__ rmean,
                                   float* __restrict__ rvar, float* __restrict__ ss,
                                   float* __restrict__ saved, long long rows, int C, float eps,
                                   float momentum) {
  __shared__ float sm[2][32][9];
  const int cl = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + cl;
  float s0 = 0.f, s1 = 0.f;
  if (c < C)
    for (int b = grp; b < nblk; b += 32) {
      s0 += partials[(long long)b * 2 * C + c];
      s1 += partials[(long long)b * 2 * C + C + c];
    }
  sm[0][grp][cl] = s0;
  sm[1][grp][cl] = s1;
  __syncthreads();
  if (grp != 0 || c >= C) return;
  s0 = s1 = 0.f;
#pragma unroll
  for (int g = 0; g < 32; ++g) {
    s0 += sm[0][g][cl];
    s1 += sm[1][g][cl];
  }
  const float inv_n = 1.0f / (float)rows;
  const float mean = s0 * inv_n;
  float var = s1 * inv_n - mean * mean;
  var = fmaxf(var, 0.f);
  const float rstd = rsqrtf(var + eps);
  const float sc = gamma[c] * rstd;
  ss[c] = sc;
  ss[C + c] = beta[c] - mean * sc;
  saved[c] = mean;
  saved[C + c] = rstd;
  if (rmean) {
    const float unbiased = rows > 1 ? var * ((float)rows / (float)(rows - 1)) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * unbiased;
  }
}

// ----------------------------------------------------------------------------- BN apply
template <bool HAS_RES, bool RES_BN>
__global__ void __launch_bounds__(kThreads, 2)
bn_apply_kernel(const void* __restrict__ y, const float* __restrict__ ss, const void* __restrict__ res,
                const float* __restrict__ rss, void* __restrict__ out, uint8_t* __restrict__ mask, long long rows, int C,
                SlabGeom gm, int act) {
  const int vpr = gm.vpr;
  const int tx = threadIdx.x % gm.tx_count;
  const int ty = threadIdx.x / gm.tx_count;
  if (tx >= vpr) return;
  float sc[8], sh[8], rsc[8], rsh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = ss[tx * 8 + i];
    sh[i] = ss[C + tx * 8 + i];
    rsc[i] = RES_BN ? rss[tx * 8 + i] : 1.f;
    rsh[i] = RES_BN ? rss[C + tx * 8 + i] : 0.f;
  }
  const long long r0 = (long long)blockIdx.x * gm.rows_per_block;
  long long r1 = r0 + gm.rows_per_block;
  if (r1 > rows) r1 = rows;
  for (long long r = r0 + ty; r < r1; r += (long long)gm.ty_count * UNROLL) {
    V8 vy[UNROLL], vr[UNROLL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const long long rr = r + (long long)u * gm.ty_count;
      ok[u] = rr < r1;
      if (ok[u]) {
        vy[u] = ldg8(y, rr * vpr + tx);
        if (HAS_RES) vr[u] = ldg8(res, rr * vpr + tx);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (!ok[u]) continue;
      float f[8];
      unpack8(vy[u], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = f[i] * sc[i] + sh[i];
      const bool res_after = (act & 8) != 0;  // DarkNet: act(bn(y)) + res; ResNet: act(bn(y) + res)
      if (res_after) {
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = act_apply(f[i], act & 7);
      }
      if (HAS_RES) {
        float rv[8];
        unpack8(vr[u], rv);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] += RES_BN ? rv[i] * rsc[i] + rsh[i] : rv[i];
      }
      if (!res_after) {
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = act_apply(f[i], act);
      }
      const long long vi = (r + (long long)u * gm.ty_count) * vpr + tx;
      const V8 o = pack8(f);
      stg8(out, vi, o);
      if (mask) {   // from the stored bf16 values, so that the mask is exactly (out > 0)
        float fo[8];
        unpack8(o, fo);
        uint32_t m = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) m |= (fo[i] > 0.f ? 1u : 0u) << i;
        mask[vi] = (uint8_t)m;
      }
    }
  }
}

// ----------------------------------------------------------------------------- BN backward apply
// dy = gamma*rstd*(g - sum_g/rows - xhat*sum_gx/rows) = A*g + B*y + K per channel
__device__ __forceinline__ void bwd_apply_coefs(const float* __restrict__ saved, const float* __restrict__ gamma,
                                                const float* __restrict__ sums, int tx, int C, float inv_rows,
                                                float (&A)[8], float (&B)[8], float (&K)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = tx * 8 + i;
    const float mean = saved[c], rstd = saved[C + c];
    const float k1 = gamma[c] * rstd;
    const float k2 = sums[c] * inv_rows, k3 = sums[C + c] * inv_rows;
    A[i] = k1;
    B[i] = -k1 * k3 * rstd;
    K[i] = -k1 * k2 + k1 * k3 * rstd * mean;
  }
}

// Mask source as in colreduce_kernel<1>: `out` (HAS_OUT), else `bits` when non-null, else recomputed from y.
template <bool HAS_OUT, bool HAS_DRES>
__global__ void __launch_bounds__(kThreads, 2)
bn_bwd_apply_kernel(const void* __restrict__ dout, const void* __restrict__ out, const uint8_t* __restrict__ bits,
                    const void* __restrict__ y, const float* __restrict__ saved, const float* __restrict__ gamma,
                    const float* __restrict__ sums, const float* __restrict__ ss, void* __restrict__ dy,
                    void* __restrict__ dres, long long rows, int C, SlabGeom gm, int act, float inv_rows) {
  const int vpr = gm.vpr;
  const int tx = threadIdx.x % gm.tx_count;
  const int ty = threadIdx.x / gm.tx_count;
  if (tx >= vpr) return;
  float A[8], B[8], K[8], sc[8], sh[8];
  const bool use_bits = !HAS_OUT && act != 0 && bits != nullptr;
  const bool recompute_mask = !HAS_OUT && act != 0 && bits == nullptr;
  bwd_apply_coefs(saved, gamma, sums, tx, C, inv_rows, A, B, K);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = recompute_mask ? ss[tx * 8 + i] : 0.f;
    sh[i] = recompute_mask ? ss[C + tx * 8 + i] : 0.f;
  }
  const long long r0 = (long long)blockIdx.x * gm.rows_per_block;
  long long r1 = r0 + gm.rows_per_block;
  if (r1 > rows) r1 = rows;
  for (long long r = r0 + ty; r < r1; r += (long long)gm.ty_count * UNROLL) {
    V8 vg[UNROLL], vo[UNROLL], vy[UNROLL];
    uint32_t mb[UNROLL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const long long rr = r + (long long)u * gm.ty_count;
      ok[u] = rr < r1;
      if (ok[u]) {
        const long long vi = rr * vpr + tx;
        vg[u] = ldg8(dout, vi);
        vy[u] = ldg8(y, vi);
        if (HAS_OUT) vo[u] = ldg8(out, vi);
        else if (use_bits) mb[u] = __ldg(bits + vi);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (!ok[u]) continue;
      const long long vi = (r + (long long)u * gm.ty_count) * vpr + tx;
      float g[8], fy[8];
      unpack8(vg[u], g);
      unpack8(vy[u], fy);
      if (HAS_OUT) {
        float fo[8];
        unpack8(vo[u], fo);
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] *= act_grad(fo[i], act);
      } else if (use_bits) {
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] *= mask_bit(mb[u], i);
      } else if (act != 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] *= act_grad(fy[i] * sc[i] + sh[i], act);
      }
      if (HAS_DRES) stg8(dres, vi, pack8(g));
      float d[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = A[i] * g[i] + B[i] * fy[i] + K[i];
      stg8(dy, vi, pack8(d));
    }
  }
}

// bn_bwd_apply_kernel for the two BatchNorms of colreduce2_kernel: dya / dyb from one read of g.  sums: [4][C] as
// folded from colreduce2_kernel's partial rows (A: sums[0..2C), B: sums[2C..4C)).
__global__ void __launch_bounds__(kThreads, 2)
bn_bwd_apply2_kernel(const void* __restrict__ g, const uint8_t* __restrict__ bits, const void* __restrict__ ya,
                     const void* __restrict__ yb, const float* __restrict__ saved_a, const float* __restrict__ saved_b,
                     const float* __restrict__ gamma_a, const float* __restrict__ gamma_b, const float* __restrict__ sums,
                     void* __restrict__ dya, void* __restrict__ dyb, long long rows, int C, SlabGeom gm, float inv_rows) {
  const int vpr = gm.vpr;
  const int tx = threadIdx.x % gm.tx_count;
  const int ty = threadIdx.x / gm.tx_count;
  if (tx >= vpr) return;
  float Aa[8], Ba[8], Ka[8], Ab[8], Bb[8], Kb[8];
  bwd_apply_coefs(saved_a, gamma_a, sums, tx, C, inv_rows, Aa, Ba, Ka);
  bwd_apply_coefs(saved_b, gamma_b, sums + 2 * C, tx, C, inv_rows, Ab, Bb, Kb);
  const long long r0 = (long long)blockIdx.x * gm.rows_per_block;
  long long r1 = r0 + gm.rows_per_block;
  if (r1 > rows) r1 = rows;
  for (long long r = r0 + ty; r < r1; r += (long long)gm.ty_count * UNROLL) {
    V8 vg[UNROLL], va[UNROLL], vb[UNROLL];
    uint32_t mk[UNROLL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const long long rr = r + (long long)u * gm.ty_count;
      ok[u] = rr < r1;
      if (ok[u]) {
        const long long vi = rr * vpr + tx;
        vg[u] = ldg8(g, vi);
        va[u] = ldg8(ya, vi);
        vb[u] = ldg8(yb, vi);
        if (bits) mk[u] = __ldg(bits + vi);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (!ok[u]) continue;
      const long long vi = (r + (long long)u * gm.ty_count) * vpr + tx;
      float fg[8], fa[8], fb[8], d[8];
      unpack8(vg[u], fg);
      unpack8(va[u], fa);
      unpack8(vb[u], fb);
      if (bits) {
#pragma unroll
        for (int i = 0; i < 8; ++i) fg[i] *= mask_bit(mk[u], i);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = Aa[i] * fg[i] + Ba[i] * fa[i] + Ka[i];
      stg8(dya, vi, pack8(d));
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = Ab[i] * fg[i] + Bb[i] * fb[i] + Kb[i];
      stg8(dyb, vi, pack8(d));
    }
  }
}

__global__ void bn_param_grad_kernel(const float* __restrict__ sums, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta, int C, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (accumulate) {
    dbeta[c] += sums[c];
    dgamma[c] += sums[C + c];
  } else {
    dbeta[c] = sums[c];
    dgamma[c] = sums[C + c];
  }
}

// ----------------------------------------------------------------------------- small elementwise
__global__ void add_bf16_kernel(void* __restrict__ a, const void* __restrict__ b, long long nvec) {
  for (long long vi = (long long)blockIdx.x * blockDim.x + threadIdx.x; vi < nvec;
       vi += (long long)gridDim.x * blockDim.x) {
    float fa[8], fb[8];
    unpack8(ldg8(a, vi), fa);
    unpack8(ldg8(b, vi), fb);
#pragma unroll
    for (int i = 0; i < 8; ++i) fa[i] += fb[i];
    stg8(a, vi, pack8(fa));
  }
}

__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}
// 8 elements per thread: two 16-byte loads, one 16-byte store (both pointers 16-byte aligned, n8 = n / 8)
__global__ void cast_bf16_vec_kernel(const float4* __restrict__ src, uint4* __restrict__ dst, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = __ldg(src + 2 * i), b = __ldg(src + 2 * i + 1);
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    dst[i] = pack8(f).q;
  }
}

__global__ void reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out, int splits,
                                       long long n, int accumulate) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float s = accumulate ? out[i] : 0.f;
    for (int k = 0; k < splits; ++k) s += partial[(long long)k * n + i];
    out[i] = s;
  }
}
// float4 variant (same summation order per element): n4 = n / 4, all pointers 16-byte aligned
__global__ void reduce_partials_vec_kernel(const float4* __restrict__ partial, float4* __restrict__ out, int splits, long long n4,
                                           int accumulate) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = accumulate ? out[i] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int k = 0; k < splits; ++k) {
      const float4 v = __ldg(partial + (long long)k * n4 + i);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    out[i] = s;
  }
}

// order 0: column (r*S+s)*Cp + c (implicit-GEMM convs, Cp = channels padded to the GEMM granule);
// order 1: column (c*R+r)*S8 + s with S8 = S rounded up to a multiple of 8 (torch order with every filter row padded
// to whole 16-byte vectors; used by the explicit im2col of 3-channel stems / patch embeddings).  Rows k >= K, channels
// c >= C and the padding columns are zero.
__global__ void prep_conv_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ o, int K, int C,
                                        int R, int S, int kpad, int order, int Kp, int Cp) {
  const long long total = (long long)Kp * kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i / kpad), j = (int)(i % kpad);
    float v = 0.f;
    if (k < K) {
      if (order == 1) {               // column (c*R + r)*S8 + s, S8 = S rounded up to 8 (matches stem_im2col_kernel)
        const int S8 = (S + 7) & ~7;
        const int cr = j / S8, sx = j % S8;
        if (cr < C * R && sx < S) v = w[(long long)k * C * R * S + (long long)cr * S + sx];
      } else if (j < R * S * Cp) {
        const int tap = j / Cp, c = j % Cp;
        if (c < C) v = w[((long long)k * C + c) * (R * S) + tap];
      }
    }
    o[i] = __float2bfloat16_rn(v);
  }
}

__global__ void finish_conv_wgrad_kernel(const float* __restrict__ partial, float* __restrict__ grad, int splits,
                                         int K, int C, int R, int S, int kpad, int accumulate, int order, int Kp,
                                         int Cp, int transposed) {
  const long long total = (long long)K * C * R * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(i % (R * S));
    const long long kc = i / (R * S);
    const int c = (int)(kc % C), k = (int)(kc / C);
    const int S8 = (S + 7) & ~7;
    const long long col = order == 1 ? (long long)(c * R + tap / S) * S8 + tap % S : (long long)tap * Cp + c;
    const long long src = transposed ? col * Kp + k : (long long)k * kpad + col;   // [Kp][kpad] or dW^T [kpad][Kp]
    float s = accumulate ? grad[i] : 0.f;
    for (int sp = 0; sp < splits; ++sp) s += partial[(long long)sp * Kp * kpad + src];
    grad[i] = s;
  }
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int C, int H,
                                    int W) {
  const long long total = (long long)N * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long hw = i % ((long long)H * W);
    const long long n = i / ((long long)H * W);
    for (int c = 0; c < C; ++c) y[i * C + c] = __float2bfloat16_rn(x[(n * C + c) * (long long)H * W + hw]);
  }
}

// Explicit im2col for 3-channel inputs (ResNet stems, ViT / SAM / VAN patch embeddings).  One block owns T consecutive
// output pixels of one output row: the (C, R, (T-1)*stride+S) input patch is staged in shared memory with coalesced
// loads; every thread then produces whole 16-byte vectors of one (pixel, channel, filter row): column
// (c*R + r)*S8 + s of the row-major [pixels][kpad] matrix (S8 = S rounded up to 8, padding columns zero), i.e. S
// consecutive floats of the staged patch per S8/8 output vectors - no per-element index table.
__global__ void __launch_bounds__(kThreads)
stem_im2col_kernel(const float* __restrict__ x, void* __restrict__ cols, int N, int C, int H, int W, int R, int S,
                   int stride, int pad, int P, int Q, int kpad, int T) {
  extern __shared__ float sm[];
  const int Wt = (T - 1) * stride + S;
  float* patch = sm;                                      // [C*R][Wt]
  const int qtiles = (Q + T - 1) / T;
  const int qt = blockIdx.x % qtiles;
  const int p = (blockIdx.x / qtiles) % P;
  const int n = blockIdx.x / (qtiles * P);
  const int q0 = qt * T;
  const int h0 = p * stride - pad, w0 = q0 * stride - pad;
  for (int i = threadIdx.x; i < C * R * Wt; i += blockDim.x) {
    const int wi = i % Wt, cr = i / Wt;
    const int r = cr % R, c = cr / R;
    const int h = h0 + r, w = w0 + wi;
    float v = 0.f;
    if (h >= 0 && h < H && w >= 0 && w < W) v = __ldg(x + (((long long)n * C + c) * H + h) * W + w);
    patch[i] = v;
  }
  __syncthreads();
  const int vpr = kpad >> 3, S8 = (S + 7) & ~7, vps = S8 >> 3;   // vectors per matrix row / per filter row
  const int npix = min(T, Q - q0);
  const long long row0 = ((long long)n * P + p) * Q + q0;
  for (int v = threadIdx.x; v < npix * vpr; v += blockDim.x) {
    const int pix = v / vpr, kv = v - pix * vpr;
    const int cr = kv / vps, s0 = (kv - cr * vps) * 8;
    float f[8];
    if (cr < C * R) {
      const float* src = patch + cr * Wt + pix * stride + s0;
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = (s0 + e < S) ? src[e] : 0.f;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = 0.f;
    }
    stg8(cols, (row0 + pix) * vpr + kv, pack8(f));
  }
}

__global__ void zero_upsample2_kernel(const void* __restrict__ dy, void* __restrict__ u, int N, int P, int Q, int H,
                                      int W, int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * H * W * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long pix = i / vpr;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    V8 val;
    val.q = make_uint4(0u, 0u, 0u, 0u);
    if (!(h & 1) && !(w & 1) && (h >> 1) < P && (w >> 1) < Q)
      val = ldg8(dy, ((n * P + (h >> 1)) * Q + (w >> 1)) * vpr + v);
    stg8(u, i, val);
  }
}

__global__ void add_strided2_kernel(void* __restrict__ dx, const void* __restrict__ dd, int N, int P, int Q, int H,
                                    int W, int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * P * Q * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long pix = i / vpr;
    const int q = (int)(pix % Q);
    const int p = (int)((pix / Q) % P);
    const long long n = pix / ((long long)Q * P);
    const long long di = ((n * H + 2 * p) * W + 2 * q) * vpr + v;
    float a[8], b[8];
    unpack8(ldg8(dx, di), a);
    unpack8(ldg8(dd, i), b);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += b[k];
    stg8(dx, di, pack8(a));
  }
}

// ----------------------------------------------------------------------------- pooling
// General K x K / stride max-pool over NHWC bf16.  Window of output (p, q) starts at
// (p*stride - pad, q*stride - pad).  Out-of-range taps are skipped (-inf padding, nn.MaxPool2d) or,
// with oob_zero, take part with the value 0 (nn.ZeroPad2d followed by an unpadded pool,
// darknet.py:212-213): their code is 255 and they receive no gradient.  argmax byte = r*K + s.
// KT > 0: the window size is a compile-time constant, so the K*K window loads are unrolled and all in flight at once
// (the runtime-K loop issues them one by one)
template <int KT>
__global__ void maxpool_fwd_kernel(const void* __restrict__ x, void* __restrict__ y, uint8_t* __restrict__ amax,
                                   int N, int H, int W, int C, int P, int Q, int Krt, int stride, int pad, int oob_zero) {
  const int K = KT > 0 ? KT : Krt;
  const int vpr = C >> 3;
  const long long total = (long long)N * P * Q * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long pix = i / vpr;
    const int q = (int)(pix % Q);
    const int p = (int)((pix / Q) % P);
    const long long n = pix / ((long long)Q * P);
    float best[8];
    int arg[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { best[k] = -INFINITY; arg[k] = 0; }
    bool first = true;
    if (KT > 0) {
      V8 win[KT > 0 ? KT * KT : 1];
      bool ok[KT > 0 ? KT * KT : 1];
#pragma unroll
      for (int r = 0; r < KT; ++r)
#pragma unroll
        for (int s = 0; s < KT; ++s) {
          const int h = stride * p - pad + r, w = stride * q - pad + s;
          ok[r * KT + s] = h >= 0 && h < H && w >= 0 && w < W;
          win[r * KT + s].zero();
          if (ok[r * KT + s]) win[r * KT + s] = ldg8(x, ((n * H + h) * W + w) * vpr + v);
        }
#pragma unroll
      for (int t = 0; t < KT * KT; ++t) {
        if (!ok[t] && !oob_zero) continue;
        float f[8];
        unpack8(win[t], f);
        const int code = ok[t] ? t : 255;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (first || f[k] > best[k]) { best[k] = f[k]; arg[k] = code; }
        first = false;
      }
    } else {
      for (int r = 0; r < K; ++r) {
        const int h = stride * p - pad + r;
        for (int s = 0; s < K; ++s) {
          const int w = stride * q - pad + s;
          const bool inside = h >= 0 && h < H && w >= 0 && w < W;
          if (!inside && !oob_zero) continue;
          float f[8];
          if (inside) {
            unpack8(ldg8(x, ((n * H + h) * W + w) * vpr + v), f);
          } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = 0.f;
          }
          const int code = inside ? r * K + s : 255;
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (first || f[k] > best[k]) { best[k] = f[k]; arg[k] = code; }
          first = false;
        }
      }
    }
    stg8(y, i, pack8(best));
    uint64_t packed = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) packed |= (uint64_t)(arg[k] & 0xff) << (8 * k);
    reinterpret_cast<uint64_t*>(amax)[i] = packed;
  }
}

// FAST: K <= 2 * stride, i.e. an input pixel lies in at most 2 x 2 output windows; the four (argmax, dy) pairs are
// loaded together instead of through two runtime-bounded loops (3x3/2 stem pool: 0.5 ms -> HBM time)
template <bool FAST>
__global__ void maxpool_bwd_kernel(const void* __restrict__ dy, const uint8_t* __restrict__ amax,
                                   void* __restrict__ dx, int N, int H, int W, int C, int P, int Q, int K, int stride,
                                   int pad) {
  const int vpr = C >> 3;
  const long long total = (long long)N * H * W * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long pix = i / vpr;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // output windows (p, q) that contain (h, w): stride*p - pad <= h <= stride*p - pad + K - 1
    const int hp = h + pad, wp = w + pad;
    const int p_hi = min(hp / stride, P - 1), q_hi = min(wp / stride, Q - 1);
    const int p_lo = max((hp - K + stride) / stride, 0), q_lo = max((wp - K + stride) / stride, 0);
    if (FAST) {
      uint64_t am[4];
      V8 gv[4];
      int code[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int p = hp / stride - (t >> 1), q = wp / stride - (t & 1);
        const int r = hp - stride * p, s2 = wp - stride * q;
        const bool ok = p >= 0 && p < P && q >= 0 && q < Q && r < K && s2 < K;
        code[t] = ok ? r * K + s2 : -1;
        am[t] = 0;
        gv[t].zero();
        if (ok) {
          const long long oi = ((n * P + p) * Q + q) * vpr + v;
          am[t] = __ldg(reinterpret_cast<const uint64_t*>(amax) + oi);
          gv[t] = ldg8(dy, oi);
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        float g[8];
        unpack8(gv[t], g);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if ((int)((am[t] >> (8 * k)) & 0xff) == code[t]) acc[k] += g[k];
      }
      stg8(dx, i, pack8(acc));
      continue;
    }
    for (int p = p_lo; p <= p_hi; ++p) {
      const int r = hp - stride * p;
      if (r < 0 || r >= K) continue;
      for (int q = q_lo; q <= q_hi; ++q) {
        const int s = wp - stride * q;
        if (s < 0 || s >= K) continue;
        const long long oi = ((n * P + p) * Q + q) * vpr + v;
        const uint64_t packed = reinterpret_cast<const uint64_t*>(amax)[oi];
        float g[8];
        unpack8(ldg8(dy, oi), g);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if ((int)((packed >> (8 * k)) & 0xff) == r * K + s) acc[k] += g[k];
      }
    }
    stg8(dx, i, pack8(acc));
  }
}

__global__ void avgpool_fwd_kernel(const void* __restrict__ x, void* __restrict__ y, int N, int HW, int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * vpr;
  const float inv = 1.f / (float)HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long n = i / vpr;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int t = 0; t < HW; ++t) {
      float f[8];
      unpack8(ldg8(x, (n * HW + t) * vpr + v), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] *= inv;
    stg8(y, i, pack8(acc));
  }
}

__global__ void avgpool_bwd_kernel(const void* __restrict__ dy, void* __restrict__ dx, int N, int HW, int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * HW * vpr;
  const float inv = 1.f / (float)HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long n = i / ((long long)HW * vpr);
    float f[8];
    unpack8(ldg8(dy, n * vpr + v), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] *= inv;
    stg8(dx, i, pack8(f));
  }
}

}  // namespace
}  // namespace saicv

using namespace saicv;

#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_version(void) { return 100; }
long long saicv_launch_count(void) { return saicv::launch_count(); }
const char* saicv_last_error(void) { return saicv::last_error(); }

int saicv_bn_stats(const void* y, float* partials, long long rows, int c, void* stream) {
  int nblk;
  return launch_colreduce<0>(y, nullptr, nullptr, nullptr, nullptr, partials, rows, c, 0, &nblk, ST);
}

int saicv_bn_finalize(const float* partials, int partial_rows_, const float* gamma, const float* beta,
                      float* running_mean, float* running_var, float* scale_shift, float* saved, long long rows,
                      int c, float eps, float momentum, void* stream) {
  const int nrows = partial_rows_ > 0 ? partial_rows_ : partial_rows(rows, c);
  bn_finalize_kernel<<<(c + 7) / 8, 256, 0, ST>>>(partials, nrows, gamma, beta, running_mean,
                                                    running_var, scale_shift, saved, rows, c, eps, momentum);
  return check_launch("bn_finalize_kernel");
}

int saicv_bn_apply(const void* y, const float* scale_shift, const void* res, const float* res_scale_shift,
                   void* out, uint32_t* mask_bits, long long rows, int c, int act, void* stream) {
  if (mask_bits && (c % 32 || (act & 7) != 1))
    return set_error("saicv_bn_apply: mask_bits needs c %% 32 == 0 and a ReLU (c=%d act=%d)", c, act);
  SlabGeom g;
  int blocks;
  if (!slab_geom(rows, c, UNROLL, &g, &blocks)) return 1;
  uint8_t* mask = reinterpret_cast<uint8_t*>(mask_bits);
  if (res == nullptr)
    bn_apply_kernel<false, false><<<blocks, kThreads, 0, ST>>>(y, scale_shift, res, res_scale_shift, out, mask, rows, c, g, act);
  else if (res_scale_shift == nullptr)
    bn_apply_kernel<true, false><<<blocks, kThreads, 0, ST>>>(y, scale_shift, res, res_scale_shift, out, mask, rows, c, g, act);
  else
    bn_apply_kernel<true, true><<<blocks, kThreads, 0, ST>>>(y, scale_shift, res, res_scale_shift, out, mask, rows, c, g, act);
  return check_launch("bn_apply_kernel");
}

// the activation-mask source of the backward kernels: `out`, the packed ReLU mask `bits`, or recomputed from y
static int check_mask_source(const char* fn, const void* out, const uint32_t* bits, const float* scale_shift, int c,
                             int act) {
  if (act != 0 && out == nullptr && bits == nullptr && scale_shift == nullptr)
    return set_error("%s: need the activated output, mask bits or scale_shift to form the activation mask", fn);
  if ((act & 7) == 3 && out != nullptr) return set_error("%s: SiLU needs the recompute path (out == NULL, scale_shift given)", fn);
  if (bits != nullptr && (act != 1 || c % 32)) return set_error("%s: mask bits need act == 1 (ReLU) and c %% 32 == 0 (c=%d)", fn, c);
  return 0;
}

int saicv_bn_bwd_reduce(const void* dout, const void* out, const uint32_t* bits, const void* y, const float* saved,
                        const float* scale_shift, float* partials, float* sums, long long rows, int c, int act,
                        void* stream) {
  if (int e = check_mask_source("saicv_bn_bwd_reduce", out, bits, scale_shift, c, act)) return e;
  int nblk;
  if (int e = launch_colreduce<1>(dout, out, y, saved, scale_shift, partials, rows, c, act, &nblk, ST, bits)) return e;
  return fold(partials, sums, nblk, 2 * c, 0, ST);
}

int saicv_bn_bwd_apply(const void* dout, const void* out, const uint32_t* bits, const void* y, const float* saved,
                       const float* gamma, const float* scale_shift, float* sums, void* dy, void* dres, float* dgamma,
                       float* dbeta, long long rows, int c, int act, int accumulate, void* stream) {
  if (int e = check_mask_source("saicv_bn_bwd_apply", out, bits, scale_shift, c, act)) return e;
  SlabGeom g;
  int blocks;
  if (!slab_geom(rows, c, UNROLL, &g, &blocks)) return 1;
  const float inv_rows = 1.0f / (float)rows;
  const uint8_t* mask = reinterpret_cast<const uint8_t*>(bits);
#define BWD_APPLY(HO, HD) \
  bn_bwd_apply_kernel<HO, HD><<<blocks, kThreads, 0, ST>>>(dout, out, mask, y, saved, gamma, sums, scale_shift, dy, dres, rows, c, g, act, inv_rows)
  if (out != nullptr && act != 0) {
    if (dres) BWD_APPLY(true, true); else BWD_APPLY(true, false);
  } else {
    if (dres) BWD_APPLY(false, true); else BWD_APPLY(false, false);
  }
#undef BWD_APPLY
  if (int e = check_launch("bn_bwd_apply_kernel")) return e;
  bn_param_grad_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sums, dgamma, dbeta, c, accumulate);
  return check_launch("bn_param_grad_kernel");
}

int saicv_bn_bwd_reduce2(const void* g, const uint32_t* bits, const void* y_a, const void* y_b, const float* saved_a,
                         const float* saved_b, float* partials, float* sums, long long rows, int c, void* stream) {
  if (bits != nullptr && c % 32) return set_error("saicv_bn_bwd_reduce2: mask bits need c %% 32 == 0 (c=%d)", c);
  SlabGeom gm;
  int nblk;
  if (!slab_geom(rows, c, 4, &gm, &nblk, kMaxPartials)) return 1;   // the geometry of launch_colreduce<1>
  colreduce2_kernel<<<nblk, kThreads, 0, ST>>>(g, reinterpret_cast<const uint8_t*>(bits), y_a, y_b, saved_a, saved_b,
                                               partials, rows, c, gm);
  if (int e = check_launch("colreduce2_kernel")) return e;
  return fold(partials, sums, nblk, 4 * c, 0, ST);
}

int saicv_bn_bwd_apply2(const void* g, const uint32_t* bits, const void* y_a, const void* y_b, const float* saved_a,
                        const float* saved_b, const float* gamma_a, const float* gamma_b, const float* sums, void* dy_a,
                        void* dy_b, float* dgamma_a, float* dbeta_a, float* dgamma_b, float* dbeta_b, long long rows,
                        int c, int accumulate_a, int accumulate_b, void* stream) {
  if (bits != nullptr && c % 32) return set_error("saicv_bn_bwd_apply2: mask bits need c %% 32 == 0 (c=%d)", c);
  SlabGeom gm;
  int blocks;
  if (!slab_geom(rows, c, UNROLL, &gm, &blocks)) return 1;
  bn_bwd_apply2_kernel<<<blocks, kThreads, 0, ST>>>(g, reinterpret_cast<const uint8_t*>(bits), y_a, y_b, saved_a,
                                                    saved_b, gamma_a, gamma_b, sums, dy_a, dy_b, rows, c, gm,
                                                    1.0f / (float)rows);
  if (int e = check_launch("bn_bwd_apply2_kernel")) return e;
  bn_param_grad_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sums, dgamma_a, dbeta_a, c, accumulate_a);
  if (int e = check_launch("bn_param_grad_kernel")) return e;
  bn_param_grad_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sums + 2 * c, dgamma_b, dbeta_b, c, accumulate_b);
  return check_launch("bn_param_grad_kernel");
}

int saicv_add_bf16(void* a, const void* b, long long n, void* stream) {
  if (n % 8) return set_error("saicv_add_bf16: n %% 8 != 0");
  add_bf16_kernel<<<grid_for(n / 8), kThreads, 0, ST>>>(a, b, n / 8);
  return check_launch("add_bf16_kernel");
}

int saicv_cast_bf16(const float* src, void* dst, long long n, void* stream) {
  if (n % 8 == 0 && ((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0) {
    cast_bf16_vec_kernel<<<grid_for(n / 8), kThreads, 0, ST>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<uint4*>(dst), n / 8);
    return check_launch("cast_bf16_vec_kernel");
  }
  cast_bf16_kernel<<<grid_for(n), kThreads, 0, ST>>>(src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  return check_launch("cast_bf16_kernel");
}

int saicv_reduce_partials(const float* partial, float* out, int splits, long long n, int accumulate,
                          void* stream) {
  if (n % 4 == 0 && ((uintptr_t)partial & 15) == 0 && ((uintptr_t)out & 15) == 0) {
    reduce_partials_vec_kernel<<<grid_for(n / 4), kThreads, 0, ST>>>(reinterpret_cast<const float4*>(partial), reinterpret_cast<float4*>(out),
                                                                    splits, n / 4, accumulate);
    return check_launch("reduce_partials_vec_kernel");
  }
  reduce_partials_kernel<<<grid_for(n), kThreads, 0, ST>>>(partial, out, splits, n, accumulate);
  return check_launch("reduce_partials_kernel");
}

int saicv_prep_conv_weight(const float* w, void* w_bf16, int k, int c, int r, int s, int kpad, int order,
                           int kp, int cp, void* stream) {
  if (kp <= 0) kp = k;
  if (cp <= 0) cp = c;
  if (kpad % 8 || kpad < r * s * (order == 1 ? c : cp) || kp < k || cp < c)
    return set_error("saicv_prep_conv_weight: bad padding (kpad %d kp %d cp %d)", kpad, kp, cp);
  prep_conv_weight_kernel<<<grid_for((long long)kp * kpad), kThreads, 0, ST>>>(
      w, reinterpret_cast<__nv_bfloat16*>(w_bf16), k, c, r, s, kpad, order, kp, cp);
  return check_launch("prep_conv_weight_kernel");
}

int saicv_finish_conv_wgrad(const float* partial, float* grad, int splits, int k, int c, int r, int s, int kpad,
                            int accumulate, int order, int kp, int cp, int transposed, void* stream) {
  if (kp <= 0) kp = k;
  if (cp <= 0) cp = c;
  finish_conv_wgrad_kernel<<<grid_for((long long)k * c * r * s), kThreads, 0, ST>>>(partial, grad, splits, k, c, r,
                                                                                     s, kpad, accumulate, order, kp, cp,
                                                                                     transposed);
  return check_launch("finish_conv_wgrad_kernel");
}

int saicv_nchw_to_nhwc_bf16(const float* x, void* y, int n, int c, int h, int w, void* stream) {
  nchw_to_nhwc_kernel<<<grid_for((long long)n * h * w), kThreads, 0, ST>>>(x, reinterpret_cast<__nv_bfloat16*>(y),
                                                                           n, c, h, w);
  return check_launch("nchw_to_nhwc_kernel");
}

int saicv_stem_kpad(int c, int r, int s) { return (c * r * ((s + 7) / 8 * 8) + 63) / 64 * 64; }

int saicv_stem_im2col(const float* x, void* cols, int n, int c, int h, int w, int r, int s, int stride, int pad,
                      int kpad, void* stream) {
  if (kpad % 8 || kpad < r * c * ((s + 7) / 8 * 8))
    return set_error("saicv_stem_im2col: kpad %d must be a multiple of 8 >= c*r*roundup(s, 8) = %d (saicv_stem_kpad)", kpad, r * c * ((s + 7) / 8 * 8));
  const int P = (h + 2 * pad - r) / stride + 1, Q = (w + 2 * pad - s) / stride + 1;
  int T = 32;  // output pixels per block; shrink until the staged patch fits in 40 KB
  while (T > 1 && ((size_t)c * r * ((T - 1) * stride + s) * 4) > 40 * 1024) T >>= 1;
  const size_t smem = (size_t)c * r * ((T - 1) * stride + s) * 4;
  if (smem > 48 * 1024) return set_error("saicv_stem_im2col: patch of %zu bytes does not fit in shared memory", smem);
  const long long blocks = (long long)n * P * ((Q + T - 1) / T);
  stem_im2col_kernel<<<(unsigned)blocks, kThreads, smem, ST>>>(x, cols, n, c, h, w, r, s, stride, pad, P, Q, kpad, T);
  return check_launch("stem_im2col_kernel");
}

int saicv_zero_upsample2(const void* dy, void* u, int n, int p, int q, int h, int w, int c, void* stream) {
  if (c % 8) return set_error("saicv_zero_upsample2: C %% 8 != 0");
  zero_upsample2_kernel<<<grid_for((long long)n * h * w * (c / 8)), kThreads, 0, ST>>>(dy, u, n, p, q, h, w, c);
  return check_launch("zero_upsample2_kernel");
}

int saicv_add_strided2(void* dx, const void* dd, int n, int p, int q, int h, int w, int c, void* stream) {
  if (c % 8) return set_error("saicv_add_strided2: C %% 8 != 0");
  add_strided2_kernel<<<grid_for((long long)n * p * q * (c / 8)), kThreads, 0, ST>>>(dx, dd, n, p, q, h, w, c);
  return check_launch("add_strided2_kernel");
}

int saicv_maxpool_fwd(const void* x, void* y, uint8_t* argmax, int n, int h, int w, int c, int k, int stride, int pad,
                      int pad_hi, int oob_zero, void* stream) {
  if (c % 8) return set_error("saicv_maxpool_fwd: C %% 8 != 0");
  if (k < 1 || k > 15 || stride < 1) return set_error("saicv_maxpool_fwd: unsupported window %d / stride %d", k, stride);
  const int P = (h + pad + pad_hi - k) / stride + 1, Q = (w + pad + pad_hi - k) / stride + 1;
  const int grid = grid_for((long long)n * P * Q * (c / 8));
  if (k == 3) maxpool_fwd_kernel<3><<<grid, kThreads, 0, ST>>>(x, y, argmax, n, h, w, c, P, Q, k, stride, pad, oob_zero);
  else if (k == 2) maxpool_fwd_kernel<2><<<grid, kThreads, 0, ST>>>(x, y, argmax, n, h, w, c, P, Q, k, stride, pad, oob_zero);
  else maxpool_fwd_kernel<0><<<grid, kThreads, 0, ST>>>(x, y, argmax, n, h, w, c, P, Q, k, stride, pad, oob_zero);
  return check_launch("maxpool_fwd_kernel");
}

int saicv_maxpool_bwd(const void* dy, const uint8_t* argmax, void* dx, int n, int h, int w, int c, int k, int stride,
                      int pad, int pad_hi, void* stream) {
  if (c % 8) return set_error("saicv_maxpool_bwd: C %% 8 != 0");
  const int P = (h + pad + pad_hi - k) / stride + 1, Q = (w + pad + pad_hi - k) / stride + 1;
  const int grid = grid_for((long long)n * h * w * (c / 8));
  if (k <= 2 * stride && k >= stride) maxpool_bwd_kernel<true><<<grid, kThreads, 0, ST>>>(dy, argmax, dx, n, h, w, c, P, Q, k, stride, pad);
  else maxpool_bwd_kernel<false><<<grid, kThreads, 0, ST>>>(dy, argmax, dx, n, h, w, c, P, Q, k, stride, pad);
  return check_launch("maxpool_bwd_kernel");
}

int saicv_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int n, int h, int w, int c, void* stream) {
  return saicv_maxpool_fwd(x, y, argmax, n, h, w, c, 3, 2, 1, 1, 0, stream);
}

int saicv_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, void* dx, int n, int h, int w, int c,
                           void* stream) {
  return saicv_maxpool_bwd(dy, argmax, dx, n, h, w, c, 3, 2, 1, 1, stream);
}

int saicv_avgpool_fwd(const void* x, void* y, int n, int hw, int c, void* stream) {
  if (c % 8) return set_error("saicv_avgpool_fwd: C %% 8 != 0");
  avgpool_fwd_kernel<<<grid_for((long long)n * (c / 8), 128), 128, 0, ST>>>(x, y, n, hw, c);
  return check_launch("avgpool_fwd_kernel");
}

int saicv_avgpool_bwd(const void* dy, void* dx, int n, int hw, int c, void* stream) {
  if (c % 8) return set_error("saicv_avgpool_bwd: C %% 8 != 0");
  avgpool_bwd_kernel<<<grid_for((long long)n * hw * (c / 8)), kThreads, 0, ST>>>(dy, dx, n, hw, c);
  return check_launch("avgpool_bwd_kernel");
}

int saicv_colsum(const void* x, float* partials, float* out, long long rows, int c, int accumulate, int is_f32,
                 void* stream) {
  if (is_f32) {
    colsum_f32_kernel<<<(c + 127) / 128, 128, 0, ST>>>(reinterpret_cast<const float*>(x), out, rows, c, accumulate);
    return check_launch("colsum_f32_kernel");
  }
  if (c % 8) return set_error("saicv_colsum: C %% 8 != 0");
  // columns are reduced in chunks of <= 2048 (the slab kernels keep one 16-byte vector per thread)
  for (int c0 = 0; c0 < c; c0 += 2048) {
    const int cw = c - c0 < 2048 ? c - c0 : 2048;
    SlabGeom g;
    int nblk;
    if (!slab_geom(rows, cw, 8, &g, &nblk, kMaxPartials)) return 1;
    g.ldv = c / 8;
    colreduce_kernel<2, 8><<<nblk, kThreads, 0, ST>>>(reinterpret_cast<const __nv_bfloat16*>(x) + c0, nullptr, nullptr,
                                                   nullptr, nullptr, nullptr, partials, rows, cw, g, 0);
    if (int e = check_launch("colreduce_kernel")) return e;
    if (int e = fold(partials, out + c0, nblk, cw, accumulate, ST)) return e;
  }
  return 0;
}

}  // extern "C"
