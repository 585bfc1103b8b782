// ViT-specific kernels of the hot path (SimpleAICV/classification/backbones/vit.py): LayerNorm
// forward/backward with the residual-stream add fused, exact-erf GELU, token assembly
// (cls + positional embedding) and token pooling.  The fused attention lives in attn_sm90.cuh / capi_attn.cu.
//
// Numerics follow the reference under autocast (SURVEY.md Appendix C): the residual stream, LayerNorm
// statistics and softmax are fp32; GEMM / attention operands are bf16 with fp32 accumulation.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "../../include/saicv_b200.h"
#include "gelu_math.cuh"
#include "host_util.h"

namespace saicv {
namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&w));
}

// ----------------------------------------------------------------------------- LayerNorm
// One warp per row; each lane owns NCH float4 chunks (columns i*128 + lane*4 .. +3).
template <int NCH>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
              __nv_bfloat16* __restrict__ y, float* __restrict__ stats, long long M, float eps) {
  constexpr int C = NCH * 128;
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  float4 g[NCH], b[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    g[i] = *reinterpret_cast<const float4*>(gamma + i * 128 + lane * 4);
    b[i] = *reinterpret_cast<const float4*>(beta + i * 128 + lane * 4);
  }
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < M; row += warps) {
    float4 v[NCH];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      v[i] = *reinterpret_cast<const float4*>(x + row * C + i * 128 + lane * 4);
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
    const float mean = warp_sum(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + bb * bb + c * c + d * d;
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + eps);
    if (lane == 0) {
      stats[row] = mean;
      stats[M + row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const uint32_t lo = pack2((v[i].x - mean) * rstd * g[i].x + b[i].x, (v[i].y - mean) * rstd * g[i].y + b[i].y);
      const uint32_t hi = pack2((v[i].z - mean) * rstd * g[i].z + b[i].z, (v[i].w - mean) * rstd * g[i].w + b[i].w);
      *reinterpret_cast<uint2*>(y + row * C + i * 128 + lane * 4) = make_uint2(lo, hi);
    }
  }
}

// dx = dres + rstd*(dxhat - mean(dxhat) - xhat*mean(dxhat*xhat)), dxhat = dy*gamma; dgamma/dbeta
// accumulated per warp in registers, folded through shared memory in a fixed order into one
// partial row per block ([gridDim.x][2][C]); ln_fold_kernel sums the rows, again in a fixed order,
// so the parameter gradients are bit-reproducible (no atomics).
template <int NCH>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ gamma,
              const float* __restrict__ stats, const float* __restrict__ dres, float* __restrict__ dx,
              __nv_bfloat16* __restrict__ dx_bf16, const float* __restrict__ row_scale, int rows_per_scale,
              float* __restrict__ partials, long long M) {
  constexpr int C = NCH * 128;
  __shared__ float red[8][C];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  float4 g[NCH], dg[NCH], db[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    g[i] = *reinterpret_cast<const float4*>(gamma + i * 128 + lane * 4);
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + warp; row < M; row += warps) {
    const float mean = stats[row], rstd = stats[M + row];
    const float bsc = row_scale ? row_scale[row / rows_per_scale] : 1.f;
    float4 xh[NCH], d[NCH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float4 xv = *reinterpret_cast<const float4*>(x + row * C + i * 128 + lane * 4);
      const uint2 dv = *reinterpret_cast<const uint2*>(dy + row * C + i * 128 + lane * 4);
      const float2 d01 = unpack2(dv.x), d23 = unpack2(dv.y);
      xh[i] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
      db[i].x += d01.x; db[i].y += d01.y; db[i].z += d23.x; db[i].w += d23.y;
      dg[i].x += d01.x * xh[i].x; dg[i].y += d01.y * xh[i].y; dg[i].z += d23.x * xh[i].z; dg[i].w += d23.y * xh[i].w;
      d[i] = make_float4(d01.x * g[i].x, d01.y * g[i].y, d23.x * g[i].z, d23.y * g[i].w);
      s1 += d[i].x + d[i].y + d[i].z + d[i].w;
      s2 += d[i].x * xh[i].x + d[i].y * xh[i].y + d[i].z * xh[i].z + d[i].w * xh[i].w;
    }
    const float c1 = warp_sum(s1) * (1.f / C), c2 = warp_sum(s2) * (1.f / C);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      float4 o = make_float4(rstd * (d[i].x - c1 - xh[i].x * c2), rstd * (d[i].y - c1 - xh[i].y * c2),
                             rstd * (d[i].z - c1 - xh[i].z * c2), rstd * (d[i].w - c1 - xh[i].w * c2));
      if (dres) {
        const float4 r = *reinterpret_cast<const float4*>(dres + row * C + i * 128 + lane * 4);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      *reinterpret_cast<float4*>(dx + row * C + i * 128 + lane * 4) = o;
      if (dx_bf16)
        *reinterpret_cast<uint2*>(dx_bf16 + row * C + i * 128 + lane * 4) =
            make_uint2(pack2(o.x * bsc, o.y * bsc), pack2(o.z * bsc, o.w * bsc));
    }
  }
  // fold the 8 warps' partial dgamma / dbeta
  for (int pass = 0; pass < 2; ++pass) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NCH; ++i)
      *reinterpret_cast<float4*>(&red[warp][i * 128 + lane * 4]) = pass == 0 ? dg[i] : db[i];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w][c];
      partials[((long long)blockIdx.x * 2 + pass) * C + c] = s;
    }
  }
}

// dgamma / dbeta (+)= sum over the per-block partial rows, fixed order: 8 columns x 32 row groups per block (the <= 264
// partial rows are spread over 32 threads per column so the fold is a handful of loads deep instead of a 264-long chain)
__global__ void ln_fold_kernel(const float* __restrict__ partials, float* __restrict__ dgamma, float* __restrict__ dbeta,
                               int nblk, int C, int accumulate) {
  __shared__ float sm[32][9];
  const int cl = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int j = blockIdx.x * 8 + cl;  // 0 .. 2C-1
  float s = 0.f;
  if (j < 2 * C)
    for (int b = grp; b < nblk; b += 32) s += partials[(long long)b * 2 * C + j];
  sm[grp][cl] = s;
  __syncthreads();
  if (grp != 0 || j >= 2 * C) return;
  float t = 0.f;
#pragma unroll
  for (int g = 0; g < 32; ++g) t += sm[g][cl];
  float* dst = j < C ? dgamma + j : dbeta + (j - C);
  *dst = accumulate ? *dst + t : t;
}

// ----------------------------------------------------------------------------- GELU (exact, erf)
// gelu_terms (gelu_math.cuh): A&S 7.1.26 erf with one ex2 and one rcp MUFU per element; libdevice erff costs ~40
// instructions per element, which made these streaming kernels compute bound.
__device__ __forceinline__ float gelu_val(float x) { return gelu_erf(x); }
__global__ void gelu_fwd_kernel(const uint4* __restrict__ u, uint4* __restrict__ h, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = u[i];
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack2(w[k]);
      w[k] = pack2(gelu_val(f.x), gelu_val(f.y));
    }
    h[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}
__device__ __forceinline__ float gelu_grad(float x) { return gelu_erf_grad(x); }
// du = dh * gelu'(u)
__global__ void gelu_bwd_kernel(const uint4* __restrict__ dh, const uint4* __restrict__ u, uint4* __restrict__ du,
                                long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 a = dh[i], b = u[i];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 d = unpack2(aw[k]), x = unpack2(bw[k]);
      o[k] = pack2(d.x * gelu_grad(x.x), d.y * gelu_grad(x.y));
    }
    du[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ----------------------------------------------------------------------------- tokens
// x[b, 0] = cls + pos[0];  x[b, 1+i] = patch[b*NP+i] + pos[1+i]      (vit.py:242-243)
__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, float* __restrict__ x, int B, int NP, int C) {
  const int c4 = C >> 2;
  const long long total = (long long)B * (NP + 1) * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4);
    const long long t = i / c4;
    const int l = (int)(t % (NP + 1));
    const long long b = t / (NP + 1);
    const float4 p = reinterpret_cast<const float4*>(pos)[(long long)l * c4 + c];
    const float4 s = l == 0 ? reinterpret_cast<const float4*>(cls)[c]
                            : reinterpret_cast<const float4*>(patch)[(b * NP + l - 1) * c4 + c];
    reinterpret_cast<float4*>(x)[i] = make_float4(s.x + p.x, s.y + p.y, s.z + p.z, s.w + p.w);
  }
}
// dpos[l] (+)= sum_b dx[b,l]; dcls (+)= sum_b dx[b,0]; dpatch[b*NP+i] = bf16(dx[b,1+i])
__global__ void assemble_tokens_bwd_kernel(const float* __restrict__ dx, float* __restrict__ dpos, float* __restrict__ dcls,
                                           __nv_bfloat16* __restrict__ dpatch, int B, int NP, int C, int accumulate) {
  const long long total = (long long)(NP + 1) * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int l = (int)(i / C);
    float s = 0.f;
    for (int b = 0; b < B; ++b) {
      const float v = dx[((long long)b * (NP + 1) + l) * C + c];
      s += v;
      if (l > 0) dpatch[((long long)b * NP + l - 1) * C + c] = __float2bfloat16_rn(v);
    }
    dpos[i] = accumulate ? dpos[i] + s : s;
    if (l == 0) dcls[c] = accumulate ? dcls[c] + s : s;
  }
}
// pooled[b] = mean over tokens 1..L-1 (global_pool, vit.py:252-255) or x[b, 0] (cls token, :258)
__global__ void token_pool_fwd_kernel(const float* __restrict__ x, float* __restrict__ pooled, int B, int L, int C, int mean_pool) {
  const long long total = (long long)B * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long b = i / C;
    if (!mean_pool) {
      pooled[i] = x[b * L * C + c];
    } else {
      float s = 0.f;
      for (int l = 1; l < L; ++l) s += x[(b * L + l) * C + c];
      pooled[i] = s / (float)(L - 1);
    }
  }
}
__global__ void token_pool_bwd_kernel(const float* __restrict__ dpooled, float* __restrict__ dx, __nv_bfloat16* __restrict__ dx_bf16,
                                      const float* __restrict__ row_scale, int B, int L, int C, int mean_pool) {
  const long long total = (long long)B * L * C;
  const float inv = 1.f / (float)(L - 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long t = i / C;
    const int l = (int)(t % L);
    const long long b = t / L;
    float v;
    if (mean_pool) v = l == 0 ? 0.f : dpooled[b * C + c] * inv;
    else v = l == 0 ? dpooled[b * C + c] : 0.f;
    dx[i] = v;
    if (dx_bf16) dx_bf16[i] = __float2bfloat16_rn(row_scale ? v * row_scale[b] : v);
  }
}

int grid_1d(long long items, int per_block = 256, int cap = 132 * 16) {
  long long b = (items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_layernorm_fwd(const float* x, const float* gamma, const float* beta, void* y, float* stats,
                        long long rows, int c, float eps, void* stream) {
  const int grid = grid_1d(rows, 8, 132 * 8);
  __nv_bfloat16* yy = reinterpret_cast<__nv_bfloat16*>(y);
  switch (c) {
    case 768: ln_fwd_kernel<6><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 1024: ln_fwd_kernel<8><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 1280: ln_fwd_kernel<10><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 512: ln_fwd_kernel<4><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 384: ln_fwd_kernel<3><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 256: ln_fwd_kernel<2><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    case 128: ln_fwd_kernel<1><<<grid, 256, 0, ST>>>(x, gamma, beta, yy, stats, rows, eps); break;
    default: return set_error("saicv_layernorm_fwd: unsupported width %d (128, 256, 384, 512, 768, 1024, 1280)", c);
  }
  return check_launch("ln_fwd_kernel");
}

int saicv_layernorm_bwd(const void* dy, const float* x, const float* gamma, const float* stats, const float* dres,
                        float* dx, void* dx_bf16, const float* bf16_row_scale, int rows_per_scale, float* partials,
                        float* dgamma, float* dbeta, long long rows, int c, int accumulate, void* stream) {
  if (bf16_row_scale && rows_per_scale <= 0) return set_error("saicv_layernorm_bwd: rows_per_scale must be > 0");
  if (!partials) return set_error("saicv_layernorm_bwd: needs a [SAICV_BN_PARTIAL_ROWS][2*c] fp32 workspace");
  const int grid = grid_1d(rows, 8 * 8, 132 * 2);
  const __nv_bfloat16* d = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* xb = reinterpret_cast<__nv_bfloat16*>(dx_bf16);
  switch (c) {
    case 768: ln_bwd_kernel<6><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 1024: ln_bwd_kernel<8><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 1280: ln_bwd_kernel<10><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 512: ln_bwd_kernel<4><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 384: ln_bwd_kernel<3><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 256: ln_bwd_kernel<2><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    case 128: ln_bwd_kernel<1><<<grid, 256, 0, ST>>>(d, x, gamma, stats, dres, dx, xb, bf16_row_scale, rows_per_scale, partials, rows); break;
    default: return set_error("saicv_layernorm_bwd: unsupported width %d", c);
  }
  if (int e = check_launch("ln_bwd_kernel")) return e;
  ln_fold_kernel<<<(2 * c + 7) / 8, 256, 0, ST>>>(partials, dgamma, dbeta, grid, c, accumulate);
  return check_launch("ln_fold_kernel");
}

int saicv_gelu_fwd(const void* u, void* h, long long n, void* stream) {
  if (n % 8) return set_error("saicv_gelu_fwd: n %% 8 != 0");
  gelu_fwd_kernel<<<grid_1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const uint4*>(u), reinterpret_cast<uint4*>(h), n / 8);
  return check_launch("gelu_fwd_kernel");
}

int saicv_gelu_bwd(const void* dh, const void* u, void* du, long long n, void* stream) {
  if (n % 8) return set_error("saicv_gelu_bwd: n %% 8 != 0");
  gelu_bwd_kernel<<<grid_1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const uint4*>(dh), reinterpret_cast<const uint4*>(u),
                                                  reinterpret_cast<uint4*>(du), n / 8);
  return check_launch("gelu_bwd_kernel");
}

int saicv_vit_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x, int b, int np, int c,
                              void* stream) {
  if (c % 4) return set_error("saicv_vit_assemble_tokens: C %% 4 != 0");
  assemble_tokens_kernel<<<grid_1d((long long)b * (np + 1) * (c / 4)), 256, 0, ST>>>(patch, cls, pos, x, b, np, c);
  return check_launch("assemble_tokens_kernel");
}

int saicv_vit_assemble_tokens_bwd(const float* dx, float* dpos, float* dcls, void* dpatch, int b, int np, int c,
                                  int accumulate, void* stream) {
  assemble_tokens_bwd_kernel<<<grid_1d((long long)(np + 1) * c), 256, 0, ST>>>(
      dx, dpos, dcls, reinterpret_cast<__nv_bfloat16*>(dpatch), b, np, c, accumulate);
  return check_launch("assemble_tokens_bwd_kernel");
}

int saicv_token_pool_fwd(const float* x, float* pooled, int b, int l, int c, int mean_pool, void* stream) {
  token_pool_fwd_kernel<<<grid_1d((long long)b * c), 256, 0, ST>>>(x, pooled, b, l, c, mean_pool);
  return check_launch("token_pool_fwd_kernel");
}

int saicv_token_pool_bwd(const float* dpooled, float* dx, void* dx_bf16, const float* bf16_row_scale, int b, int l,
                         int c, int mean_pool, void* stream) {
  token_pool_bwd_kernel<<<grid_1d((long long)b * l * c), 256, 0, ST>>>(dpooled, dx, reinterpret_cast<__nv_bfloat16*>(dx_bf16),
                                                                       bf16_row_scale, b, l, c, mean_pool);
  return check_launch("token_pool_bwd_kernel");
}

}  // extern "C"
