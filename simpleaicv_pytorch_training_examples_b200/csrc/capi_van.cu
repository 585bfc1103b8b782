// HBM / L1-bound kernels of the VAN and ConvFormer hot paths (SimpleAICV/classification/backbones/van.py,
// convformer.py): depthwise convolutions (3x3, 5x5, 7x7 dilation 3; :20-35,59-93; ConvFormer's 7x7 with the
// ReLU-masked data gradient) forward / data gradient / weight gradient, the global average pool of an fp32 or
// bf16 stream (convformer.py:251-254), the LKA
// gating multiply (:91), the layer-scale residual update (:183-184), BatchNorm over an fp32 residual stream
// (:160-165,205-207) and a generic NHWC im2col for the strided patch-embedding convolutions (:189-208).
// Activations are NHWC bf16 seen as [rows][C]; the residual stream is fp32 (the reference's dtype flow under
// autocast: fp32 layer-scale parameter * bf16 branch promotes the sum to fp32).  Every reduction is two-stage
// with a fixed order (bit-reproducible, no atomics).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"
#include "vec8.cuh"

namespace saicv {
namespace {

// 8 consecutive elements starting at element index `e` of a bf16 or fp32 tensor
__device__ __forceinline__ void load8(const void* p, long long e, bool f32, float (&f)[8]) {
  if (f32) {
    const float4 a = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + e);
    const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + e + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    unpack8(*reinterpret_cast<const V8*>(reinterpret_cast<const __nv_bfloat16*>(p) + e), f);
  }
}
__device__ __forceinline__ void store8(void* p, long long e, bool f32, const float (&f)[8]) {
  if (f32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p) + e) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p) + e + 4) = make_float4(f[4], f[5], f[6], f[7]);
  } else {
    *reinterpret_cast<V8*>(reinterpret_cast<__nv_bfloat16*>(p) + e) = pack8(f);
  }
}

// ----------------------------------------------------------------------------- depthwise convolution
// Block = 32 pixels x 8 channel vectors (64 channels); blockIdx.y = 64-channel chunk; the chunk's K*K*64
// weights sit in shared memory as [tap][64] fp32.  flip: taps mirrored (data gradient of a 'same' conv).
// MASK (compile-time, appended parameter unused otherwise): y *= (mask > 0) with mask bf16 of y's shape, the
// ReLU in FRONT of the conv (convformer.py:65-70: dwconv(relu(pwconv1(x)))) applied to its data gradient.
template <int K, bool MASK = false>
__global__ void __launch_bounds__(256)
dwconv_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
              __nv_bfloat16* __restrict__ y, int N, int H, int W, int C, int dil, int relu, int flip,
              const __nv_bfloat16* __restrict__ mask = nullptr) {
  constexpr int KK = K * K;
  __shared__ float sw[KK][64];
  __shared__ float sb[64];
  const int c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < KK * 64; i += 256) {
    const int tap = i / 64, c = i % 64;
    const int src_tap = flip ? KK - 1 - tap : tap;
    sw[tap][c] = (c0 + c < C) ? w[(long long)(c0 + c) * KK + src_tap] : 0.f;   // torch layout [C][1][K][K]
  }
  if (threadIdx.x < 64) sb[threadIdx.x] = (bias && c0 + threadIdx.x < C) ? bias[c0 + threadIdx.x] : 0.f;
  __syncthreads();
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c = c0 + cv * 8;
  if (c >= C) return;
  const int pad = dil * (K - 1) / 2;
  const long long npix = (long long)N * H * W;
  for (long long pix = (long long)blockIdx.x * 32 + pl; pix < npix; pix += (long long)gridDim.x * 32) {
    const int wq = (int)(pix % W);
    const int hq = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = sb[cv * 8 + i];
#pragma unroll
    for (int r = 0; r < K; ++r) {
      const int hh = hq + r * dil - pad;
      if (hh < 0 || hh >= H) continue;
#pragma unroll
      for (int s = 0; s < K; ++s) {
        const int ww = wq + s * dil - pad;
        if (ww < 0 || ww >= W) continue;
        float f[8];
        unpack8(*reinterpret_cast<const V8*>(x + ((n * H + hh) * W + ww) * C + c), f);
        const float* wt = &sw[r * K + s][cv * 8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(f[i], wt[i], acc[i]);
      }
    }
    if (relu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaxf(acc[i], 0.f);
    }
    if (MASK) {
      float m[8];
      unpack8(*reinterpret_cast<const V8*>(mask + pix * C + c), m);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = m[i] > 0.f ? acc[i] : 0.f;
    }
    *reinterpret_cast<V8*>(y + pix * C + c) = pack8(acc);
  }
}

// dw[c][r][s] = sum_pixels dy[pix][c] * x[pix shifted by the tap][c].  Block (slab of pixels, 64-channel chunk):
// every thread keeps 8 channel sums for ONE tap at a time; partial[blockIdx.x][tap][C].
template <int K>
__global__ void __launch_bounds__(256)
dwconv_wgrad_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, float* __restrict__ partial,
                    int N, int H, int W, int C, int dil, long long pix_per_block) {
  constexpr int KK = K * K;
  __shared__ float red[32][65];
  const int c0 = blockIdx.y * 64;
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c = c0 + cv * 8;
  const bool live = c < C;
  const int pad = dil * (K - 1) / 2;
  const long long npix = (long long)N * H * W;
  const long long p0 = (long long)blockIdx.x * pix_per_block;
  const long long p1 = min(npix, p0 + pix_per_block);
  for (int tap = 0; tap < KK; ++tap) {
    const int r = tap / K, s = tap % K;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if (live) {
      for (long long pix = p0 + pl; pix < p1; pix += 32) {
        const int wq = (int)(pix % W);
        const int hq = (int)((pix / W) % H);
        const long long n = pix / ((long long)W * H);
        const int hh = hq + r * dil - pad, ww = wq + s * dil - pad;
        if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
        float g[8], f[8];
        unpack8(*reinterpret_cast<const V8*>(dy + pix * C + c), g);
        unpack8(*reinterpret_cast<const V8*>(x + ((n * H + hh) * W + ww) * C + c), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(g[i], f[i], acc[i]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) red[pl][cv * 8 + i] = acc[i];
    __syncthreads();
    if (threadIdx.x < 64 && c0 + threadIdx.x < C) {
      float t = 0.f;
#pragma unroll 8
      for (int q = 0; q < 32; ++q) t += red[q][threadIdx.x];
      partial[((long long)blockIdx.x * KK + tap) * C + c0 + threadIdx.x] = t;
    }
  }
}
// grad[c][tap] (+)= sum_b partial[b][tap][c]
__global__ void dwconv_wgrad_fold_kernel(const float* __restrict__ partial, float* __restrict__ grad, int nblk, int KK, int C,
                                         int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KK * C) return;
  const int c = i / KK, tap = i % KK;
  float s = 0.f;
  for (int b = 0; b < nblk; ++b) s += partial[((long long)b * KK + tap) * C + c];
  grad[i] = accumulate ? grad[i] + s : s;
}

// ----------------------------------------------------------------------------- global average pool of a stream
// y[n][c] = bf16(sum_t x[n][t][c] * (1 / HW)), x bf16 or fp32, summed in fp32 in t order (the reference pools the
// stream in its own dtype and autocast casts the pooled features for the head Linear, convformer.py:251-254)
__global__ void avgpool_stream_fwd_kernel(const void* __restrict__ x, int x_f32, __nv_bfloat16* __restrict__ y, int N, int HW,
                                          int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * vpr;
  const float inv = 1.f / (float)HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long n = i / vpr;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int t = 0; t < HW; ++t) {
      float f[8];
      load8(x, ((n * HW + t) * vpr + v) * 8, x_f32 != 0, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] *= inv;
    store8(y, i * 8, false, acc);
  }
}
// dx[n][t][c] = dy[n][c] * (1 / HW), dy bf16, dx fp32 or bf16
__global__ void avgpool_stream_bwd_kernel(const __nv_bfloat16* __restrict__ dy, void* __restrict__ dx, int dx_f32, int N, int HW,
                                          int C) {
  const int vpr = C >> 3;
  const long long total = (long long)N * HW * vpr;
  const float inv = 1.f / (float)HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long n = i / ((long long)HW * vpr);
    float f[8];
    load8(dy, (n * vpr + v) * 8, false, f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] *= inv;
    store8(dx, i * 8, dx_f32 != 0, f);
  }
}

// ----------------------------------------------------------------------------- elementwise
// out = a * b
__global__ void mul_kernel(const V8* __restrict__ a, const V8* __restrict__ b, V8* __restrict__ out, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(a[i], x);
    unpack8(b[i], y);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] *= y[k];
    out[i] = pack8(x);
  }
}
// out = (dg * c1 + dlk) * (p1 > 0)      (gradient reaching the ReLU output p1 from the gate and from the LKA convs)
__global__ void gate_bwd_kernel(const V8* __restrict__ dg, const V8* __restrict__ c1, const V8* __restrict__ dlk,
                                const V8* __restrict__ p1, V8* __restrict__ out, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8], c[8], d[8];
    unpack8(dg[i], a);
    unpack8(c1[i], b);
    unpack8(dlk[i], c);
    unpack8(p1[i], d);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = d[k] > 0.f ? fmaf(a[k], b[k], c[k]) : 0.f;
    out[i] = pack8(a);
  }
}

// x_out = x + rs[row / rows_per_scale] * ls[c] * (branch [+ shortcut])         (fp32 residual stream)
__global__ void ls_residual_fwd_kernel(const void* __restrict__ x, int x_f32, const __nv_bfloat16* __restrict__ br,
                                       const __nv_bfloat16* __restrict__ sc, const float* __restrict__ ls,
                                       const float* __restrict__ rs, int rows_per_scale, float* __restrict__ out, long long rows,
                                       int C) {
  const int vpr = C >> 3;
  const long long total = rows * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long row = i / vpr;
    const float s = rs ? rs[row / rows_per_scale] : 1.f;
    float xv[8], b[8];
    load8(x, i * 8, x_f32 != 0, xv);
    load8(br, i * 8, false, b);
    if (sc) {
      float t[8];
      load8(sc, i * 8, false, t);
#pragma unroll
      for (int k = 0; k < 8; ++k) b[k] += t[k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) xv[k] = fmaf(s * ls[v * 8 + k], b[k], xv[k]);
    store8(out, i * 8, true, xv);
  }
}
// dy = rs * ls[c] * dxn (bf16);  partial[blk][c] = sum_rows rs * dxn * (branch [+ shortcut])
__global__ void __launch_bounds__(256)
ls_residual_bwd_kernel(const float* __restrict__ dxn, const __nv_bfloat16* __restrict__ br, const __nv_bfloat16* __restrict__ sc,
                       const float* __restrict__ ls, const float* __restrict__ rs, int rows_per_scale,
                       __nv_bfloat16* __restrict__ dy, float* __restrict__ partial, long long rows, int C, int tx_count,
                       long long rows_per_block) {
  __shared__ float red[256][9];
  const int vpr = C >> 3;
  const int tx = threadIdx.x % tx_count, ty = threadIdx.x / tx_count, ty_count = 256 / tx_count;
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (int v = tx; v < ((vpr + tx_count - 1) / tx_count) * tx_count; v += tx_count) {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    if (v < vpr) {
      float lsv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) lsv[k] = ls[v * 8 + k];
      for (long long row = r0 + ty; row < r1; row += ty_count) {
        const float s = rs ? rs[row / rows_per_scale] : 1.f;
        const long long e = (row * vpr + v) * 8;
        float g[8], b[8], o[8];
        load8(dxn, e, true, g);
        load8(br, e, false, b);
        if (sc) {
          float t[8];
          load8(sc, e, false, t);
#pragma unroll
          for (int k = 0; k < 8; ++k) b[k] += t[k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          o[k] = s * lsv[k] * g[k];
          acc[k] = fmaf(s * g[k], b[k], acc[k]);
        }
        store8(dy, e, false, o);
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.x][k] = acc[k];
    __syncthreads();
    if (ty == 0 && v < vpr) {
      float t[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) t[k] = 0.f;
      for (int q = 0; q < ty_count; ++q)
#pragma unroll
        for (int k = 0; k < 8; ++k) t[k] += red[q * tx_count + tx][k];
#pragma unroll
      for (int k = 0; k < 8; ++k) partial[(long long)blockIdx.x * C + v * 8 + k] = t[k];
    }
  }
}

// ----------------------------------------------------------------------------- BatchNorm, generic dtypes
// MODE 0: partial[blk][0][c] = sum x, [1][c] = sum x^2                 (forward statistics)
// MODE 1: partial[blk][0][c] = sum g, [1][c] = sum g * xhat           (backward reductions)
template <int MODE>
__global__ void __launch_bounds__(256)
bn_colreduce_generic_kernel(const void* __restrict__ x, int x_f32, const void* __restrict__ g, int g_f32,
                            const float* __restrict__ saved, float* __restrict__ partial, long long rows, int C, int tx_count,
                            long long rows_per_block) {
  __shared__ float red[256][17];
  const int vpr = C >> 3;
  const int tx = threadIdx.x % tx_count, ty = threadIdx.x / tx_count, ty_count = 256 / tx_count;
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (int v = tx; v < ((vpr + tx_count - 1) / tx_count) * tx_count; v += tx_count) {
    float s0[8], s1[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s0[k] = s1[k] = 0.f;
    if (v < vpr) {
      float mean[8], rstd[8];
      if (MODE == 1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          mean[k] = saved[v * 8 + k];
          rstd[k] = saved[C + v * 8 + k];
        }
      }
      for (long long row = r0 + ty; row < r1; row += ty_count) {
        const long long e = (row * vpr + v) * 8;
        float xv[8];
        load8(x, e, x_f32 != 0, xv);
        if (MODE == 0) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            s0[k] += xv[k];
            s1[k] = fmaf(xv[k], xv[k], s1[k]);
          }
        } else {
          float gv[8];
          load8(g, e, g_f32 != 0, gv);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            s0[k] += gv[k];
            s1[k] = fmaf(gv[k], (xv[k] - mean[k]) * rstd[k], s1[k]);
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      red[threadIdx.x][k] = s0[k];
      red[threadIdx.x][8 + k] = s1[k];
    }
    __syncthreads();
    if (ty == 0 && v < vpr) {
      float t[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) t[k] = 0.f;
      for (int q = 0; q < ty_count; ++q)
#pragma unroll
        for (int k = 0; k < 16; ++k) t[k] += red[q * tx_count + tx][k];
      float* prow = partial + (long long)blockIdx.x * 2 * C;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        prow[v * 8 + k] = t[k];
        prow[C + v * 8 + k] = t[8 + k];
      }
    }
  }
}
// out = x * scale + shift
__global__ void bn_apply_generic_kernel(const void* __restrict__ x, int x_f32, const float* __restrict__ ss, void* __restrict__ out,
                                        int out_f32, long long rows, int C) {
  const int vpr = C >> 3;
  const long long total = rows * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    float f[8];
    load8(x, i * 8, x_f32 != 0, f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = fmaf(f[k], ss[v * 8 + k], ss[C + v * 8 + k]);
    store8(out, i * 8, out_f32 != 0, f);
  }
}
// dx = gamma*rstd*(g - sum_g/rows - xhat*sum_gx/rows) [+ dres]
__global__ void bn_bwd_apply_generic_kernel(const void* __restrict__ x, int x_f32, const void* __restrict__ g, int g_f32,
                                            const float* __restrict__ saved, const float* __restrict__ gamma,
                                            const float* __restrict__ sums, const float* __restrict__ dres, void* __restrict__ dx,
                                            int dx_f32, long long rows, int C, float inv_rows) {
  const int vpr = C >> 3;
  const long long total = rows * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    float xv[8], gv[8], o[8];
    load8(x, i * 8, x_f32 != 0, xv);
    load8(g, i * 8, g_f32 != 0, gv);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = v * 8 + k;
      const float mean = saved[c], rstd = saved[C + c];
      const float k1 = gamma[c] * rstd;
      const float xh = (xv[k] - mean) * rstd;
      o[k] = k1 * (gv[k] - sums[c] * inv_rows - xh * sums[C + c] * inv_rows);
    }
    if (dres) {
      float r[8];
      load8(dres, i * 8, true, r);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] += r[k];
    }
    store8(dx, i * 8, dx_f32 != 0, o);
  }
}
__global__ void bn_param_grad_generic_kernel(const float* __restrict__ sums, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                             int C, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  dbeta[c] = accumulate ? dbeta[c] + sums[c] : sums[c];
  dgamma[c] = accumulate ? dgamma[c] + sums[C + c] : sums[C + c];
}

// ----------------------------------------------------------------------------- NHWC im2col / col2im
// cols[(n*P+p)*Q+q][(r*S+s)*C + c] = x[n][p*stride-pad+r][q*stride-pad+s][c]   (0 outside)
__global__ void im2col_nhwc_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ cols, int N, int H, int W, int C,
                                   int K, int stride, int pad, int P, int Q) {
  const int vpr = C >> 3;
  const long long total = (long long)N * P * Q * K * K * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int tap = (int)(t % (K * K));
    t /= K * K;
    const int q = (int)(t % Q);
    const int p = (int)((t / Q) % P);
    const long long n = t / ((long long)Q * P);
    const int h = p * stride - pad + tap / K, w = q * stride - pad + tap % K;
    V8 val;
    val.zero();
    if (h >= 0 && h < H && w >= 0 && w < W) val = *reinterpret_cast<const V8*>(x + ((n * H + h) * W + w) * C + v * 8);
    *reinterpret_cast<V8*>(cols + i * 8) = val;
  }
}
// dx[n][h][w][c] = sum over (p, q, tap) that read it of dcols[...]     (gather form: deterministic)
__global__ void col2im_nhwc_kernel(const __nv_bfloat16* __restrict__ dcols, __nv_bfloat16* __restrict__ dx, int N, int H, int W,
                                   int C, int K, int stride, int pad, int P, int Q) {
  const int vpr = C >> 3;
  const long long total = (long long)N * H * W * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long pix = i / vpr;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int r = 0; r < K; ++r) {
      const int hp = h + pad - r;
      if (hp < 0 || hp % stride) continue;
      const int p = hp / stride;
      if (p >= P) continue;
      for (int s = 0; s < K; ++s) {
        const int wp = w + pad - s;
        if (wp < 0 || wp % stride) continue;
        const int q = wp / stride;
        if (q >= Q) continue;
        float f[8];
        unpack8(*reinterpret_cast<const V8*>(dcols + ((((n * P + p) * Q + q) * K * K + r * K + s) * vpr + v) * 8), f);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += f[k];
      }
    }
    *reinterpret_cast<V8*>(dx + i * 8) = pack8(acc);
  }
}

int grid1d(long long items, int per_block = 256, int cap = 132 * 16) {
  long long b = (items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}
int pow2_ge(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}
// slab geometry of the column reductions: tx_count threads across 8-column vectors, rows split over <= 264 blocks
void slab(long long rows, int C, int* tx_count, long long* rows_per_block, int* nblk) {
  const int vpr = C / 8;
  int tx = pow2_ge(vpr);
  if (tx > 256) tx = 256;
  const int ty = 256 / tx;
  long long b = (rows + (long long)ty * 8 - 1) / ((long long)ty * 8);
  if (b > SAICV_BN_PARTIAL_ROWS) b = SAICV_BN_PARTIAL_ROWS;
  if (b < 1) b = 1;
  long long rpb = (rows + b - 1) / b;
  rpb = (rpb + ty - 1) / ty * ty;
  *tx_count = tx;
  *rows_per_block = rpb;
  *nblk = (int)((rows + rpb - 1) / rpb);
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_dwconv_fwd(const void* x, const float* w, const float* bias, void* y, int n, int h, int wd, int c, int k, int dil,
                     int relu, int flip, void* stream) {
  if (c % 8) return set_error("saicv_dwconv_fwd: C %% 8 != 0");
  const long long npix = (long long)n * h * wd;
  dim3 grid((unsigned)grid1d(npix, 32, 132 * 8), (unsigned)((c + 63) / 64));
  const __nv_bfloat16* xx = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* yy = reinterpret_cast<__nv_bfloat16*>(y);
  switch (k) {
    case 3: dwconv_kernel<3><<<grid, 256, 0, ST>>>(xx, w, bias, yy, n, h, wd, c, dil, relu, flip); break;
    case 5: dwconv_kernel<5><<<grid, 256, 0, ST>>>(xx, w, bias, yy, n, h, wd, c, dil, relu, flip); break;
    case 7: dwconv_kernel<7><<<grid, 256, 0, ST>>>(xx, w, bias, yy, n, h, wd, c, dil, relu, flip); break;
    default: return set_error("saicv_dwconv_fwd: kernel size %d (3, 5, 7)", k);
  }
  return check_launch("dwconv_kernel");
}

int saicv_dwconv_dgrad_masked(const void* dy, const float* w, const void* mask, void* dx, int n, int h, int wd, int c, int k,
                              void* stream) {
  if (c % 8) return set_error("saicv_dwconv_dgrad_masked: C %% 8 != 0");
  if (!mask) return set_error("saicv_dwconv_dgrad_masked: mask is NULL");
  if (k != 7) return set_error("saicv_dwconv_dgrad_masked: kernel size %d (7)", k);
  const long long npix = (long long)n * h * wd;
  dim3 grid((unsigned)grid1d(npix, 32, 132 * 8), (unsigned)((c + 63) / 64));
  dwconv_kernel<7, true><<<grid, 256, 0, ST>>>(reinterpret_cast<const __nv_bfloat16*>(dy), w, nullptr,
                                               reinterpret_cast<__nv_bfloat16*>(dx), n, h, wd, c, 1, 0, 1,
                                               reinterpret_cast<const __nv_bfloat16*>(mask));
  return check_launch("dwconv_kernel");
}

int saicv_avgpool_stream_fwd(const void* x, int x_f32, void* y, int n, int hw, int c, void* stream) {
  if (c % 8) return set_error("saicv_avgpool_stream_fwd: C %% 8 != 0");
  avgpool_stream_fwd_kernel<<<grid1d((long long)n * (c / 8), 128), 128, 0, ST>>>(x, x_f32, reinterpret_cast<__nv_bfloat16*>(y), n,
                                                                                 hw, c);
  return check_launch("avgpool_stream_fwd_kernel");
}

int saicv_avgpool_stream_bwd(const void* dy, void* dx, int dx_f32, int n, int hw, int c, void* stream) {
  if (c % 8) return set_error("saicv_avgpool_stream_bwd: C %% 8 != 0");
  avgpool_stream_bwd_kernel<<<grid1d((long long)n * hw * (c / 8)), 256, 0, ST>>>(reinterpret_cast<const __nv_bfloat16*>(dy), dx,
                                                                                 dx_f32, n, hw, c);
  return check_launch("avgpool_stream_bwd_kernel");
}

int saicv_dwconv_wgrad_blocks(long long npix) {
  long long b = (npix + 255) / 256;
  if (b > 132) b = 132;
  return (int)(b < 1 ? 1 : b);
}

int saicv_dwconv_wgrad(const void* dy, const void* x, float* partial, float* dw, int n, int h, int wd, int c, int k, int dil,
                       int accumulate, void* stream) {
  if (c % 8) return set_error("saicv_dwconv_wgrad: C %% 8 != 0");
  const long long npix = (long long)n * h * wd;
  const int nblk = saicv_dwconv_wgrad_blocks(npix);
  const long long ppb = (npix + nblk - 1) / nblk;
  dim3 grid((unsigned)nblk, (unsigned)((c + 63) / 64));
  const __nv_bfloat16* g = reinterpret_cast<const __nv_bfloat16*>(dy);
  const __nv_bfloat16* xx = reinterpret_cast<const __nv_bfloat16*>(x);
  switch (k) {
    case 3: dwconv_wgrad_kernel<3><<<grid, 256, 0, ST>>>(g, xx, partial, n, h, wd, c, dil, ppb); break;
    case 5: dwconv_wgrad_kernel<5><<<grid, 256, 0, ST>>>(g, xx, partial, n, h, wd, c, dil, ppb); break;
    case 7: dwconv_wgrad_kernel<7><<<grid, 256, 0, ST>>>(g, xx, partial, n, h, wd, c, dil, ppb); break;
    default: return set_error("saicv_dwconv_wgrad: kernel size %d (3, 5, 7)", k);
  }
  if (int e = check_launch("dwconv_wgrad_kernel")) return e;
  dwconv_wgrad_fold_kernel<<<(k * k * c + 255) / 256, 256, 0, ST>>>(partial, dw, nblk, k * k, c, accumulate);
  return check_launch("dwconv_wgrad_fold_kernel");
}

int saicv_mul_bf16(const void* a, const void* b, void* out, long long n, void* stream) {
  if (n % 8) return set_error("saicv_mul_bf16: n %% 8 != 0");
  mul_kernel<<<grid1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const V8*>(a), reinterpret_cast<const V8*>(b), reinterpret_cast<V8*>(out), n / 8);
  return check_launch("mul_kernel");
}

int saicv_gate_bwd(const void* dg, const void* c1, const void* dlk, const void* p1, void* out, long long n, void* stream) {
  if (n % 8) return set_error("saicv_gate_bwd: n %% 8 != 0");
  gate_bwd_kernel<<<grid1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const V8*>(dg), reinterpret_cast<const V8*>(c1),
                                                 reinterpret_cast<const V8*>(dlk), reinterpret_cast<const V8*>(p1),
                                                 reinterpret_cast<V8*>(out), n / 8);
  return check_launch("gate_bwd_kernel");
}

int saicv_ls_residual_fwd(const void* x, int x_f32, const void* branch, const void* shortcut, const float* ls, const float* row_scale,
                          int rows_per_scale, float* out, long long rows, int c, void* stream) {
  if (c % 8) return set_error("saicv_ls_residual_fwd: C %% 8 != 0");
  if (row_scale && rows_per_scale <= 0) return set_error("saicv_ls_residual_fwd: rows_per_scale must be > 0");
  ls_residual_fwd_kernel<<<grid1d(rows * (c / 8)), 256, 0, ST>>>(x, x_f32, reinterpret_cast<const __nv_bfloat16*>(branch),
                                                                 reinterpret_cast<const __nv_bfloat16*>(shortcut), ls, row_scale,
                                                                 rows_per_scale, out, rows, c);
  return check_launch("ls_residual_fwd_kernel");
}

int saicv_ls_residual_bwd(const float* dxn, const void* branch, const void* shortcut, const float* ls, const float* row_scale,
                          int rows_per_scale, void* dy, float* partial, float* dls, long long rows, int c, int accumulate,
                          void* stream) {
  if (c % 8) return set_error("saicv_ls_residual_bwd: C %% 8 != 0");
  int tx, nblk;
  long long rpb;
  slab(rows, c, &tx, &rpb, &nblk);
  ls_residual_bwd_kernel<<<nblk, 256, 0, ST>>>(dxn, reinterpret_cast<const __nv_bfloat16*>(branch),
                                               reinterpret_cast<const __nv_bfloat16*>(shortcut), ls, row_scale, rows_per_scale,
                                               reinterpret_cast<__nv_bfloat16*>(dy), partial, rows, c, tx, rpb);
  if (int e = check_launch("ls_residual_bwd_kernel")) return e;
  return saicv_reduce_partials(partial, dls, nblk, c, accumulate, stream);
}

int saicv_bn_stats_generic(const void* x, int x_f32, float* partial, long long rows, int c, void* stream) {
  if (c % 8) return set_error("saicv_bn_stats_generic: C %% 8 != 0");
  int tx, nblk;
  long long rpb;
  slab(rows, c, &tx, &rpb, &nblk);
  bn_colreduce_generic_kernel<0><<<nblk, 256, 0, ST>>>(x, x_f32, nullptr, 0, nullptr, partial, rows, c, tx, rpb);
  if (int e = check_launch("bn_colreduce_generic_kernel")) return e;
  return nblk > 0 ? 0 : 1;
}
int saicv_bn_generic_partial_rows(long long rows, int c) {
  int tx, nblk;
  long long rpb;
  slab(rows, c, &tx, &rpb, &nblk);
  return nblk;
}

int saicv_bn_apply_generic(const void* x, int x_f32, const float* scale_shift, void* out, int out_f32, long long rows, int c,
                           void* stream) {
  if (c % 8) return set_error("saicv_bn_apply_generic: C %% 8 != 0");
  bn_apply_generic_kernel<<<grid1d(rows * (c / 8)), 256, 0, ST>>>(x, x_f32, scale_shift, out, out_f32, rows, c);
  return check_launch("bn_apply_generic_kernel");
}

int saicv_bn_bwd_generic(const void* x, int x_f32, const void* g, int g_f32, const float* saved, const float* gamma,
                         const float* dres, float* partial, float* sums, void* dx, int dx_f32, float* dgamma, float* dbeta,
                         long long rows, int c, int accumulate, void* stream) {
  if (c % 8) return set_error("saicv_bn_bwd_generic: C %% 8 != 0");
  int tx, nblk;
  long long rpb;
  slab(rows, c, &tx, &rpb, &nblk);
  bn_colreduce_generic_kernel<1><<<nblk, 256, 0, ST>>>(x, x_f32, g, g_f32, saved, partial, rows, c, tx, rpb);
  if (int e = check_launch("bn_colreduce_generic_kernel")) return e;
  if (int e = saicv_reduce_partials(partial, sums, nblk, 2LL * c, 0, stream)) return e;
  bn_bwd_apply_generic_kernel<<<grid1d(rows * (c / 8)), 256, 0, ST>>>(x, x_f32, g, g_f32, saved, gamma, sums, dres, dx, dx_f32,
                                                                      rows, c, 1.0f / (float)rows);
  if (int e = check_launch("bn_bwd_apply_generic_kernel")) return e;
  bn_param_grad_generic_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sums, dgamma, dbeta, c, accumulate);
  return check_launch("bn_param_grad_generic_kernel");
}

int saicv_im2col_nhwc(const void* x, void* cols, int n, int h, int w, int c, int k, int stride, int pad, void* stream) {
  if (c % 8) return set_error("saicv_im2col_nhwc: C %% 8 != 0");
  const int P = (h + 2 * pad - k) / stride + 1, Q = (w + 2 * pad - k) / stride + 1;
  im2col_nhwc_kernel<<<grid1d((long long)n * P * Q * k * k * (c / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(cols), n, h, w, c, k, stride, pad, P, Q);
  return check_launch("im2col_nhwc_kernel");
}

int saicv_col2im_nhwc(const void* dcols, void* dx, int n, int h, int w, int c, int k, int stride, int pad, void* stream) {
  if (c % 8) return set_error("saicv_col2im_nhwc: C %% 8 != 0");
  const int P = (h + 2 * pad - k) / stride + 1, Q = (w + 2 * pad - k) / stride + 1;
  col2im_nhwc_kernel<<<grid1d((long long)n * h * w * (c / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(dcols), reinterpret_cast<__nv_bfloat16*>(dx), n, h, w, c, k, stride, pad, P, Q);
  return check_launch("col2im_nhwc_kernel");
}

}  // extern "C"
