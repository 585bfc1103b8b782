// DETR transformer glue kernels (SimpleAICV/detection/models/detr.py:44-180): post-LayerNorm on the fp32
// token stream with the bf16 GEMM-operand copies (y and y + positional embedding) written by the same pass,
// its backward, the counter-hash dropout used by the residual / feed-forward dropouts, and the packing of
// projected q / k rows into the per-head [B, H, L, DP] score operands (with one extra column that carries the
// additive key bias of nn.MultiheadAttention's float key_padding_mask).  All are HBM-bound streaming kernels:
// one warp per row for the LayerNorms, 16-byte vectors elsewhere.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "dropout_hash.cuh"
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
__device__ __forceinline__ void st_bf16x4(__nv_bfloat16* p, float4 v) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack2(v.x, v.y), pack2(v.z, v.w));
}

// ----------------------------------------------------------------------------- post-LN forward
// y = LN(z) (fp32 stream); yb = bf16(y); ypb = bf16(y + pos[row % pos_rows]).  One warp per row.
template <int NCH>
__global__ void __launch_bounds__(256)
postln_fwd_kernel(const float* __restrict__ z, const float* __restrict__ gamma, const float* __restrict__ beta,
                  float* __restrict__ y, __nv_bfloat16* __restrict__ yb, const float* __restrict__ pos, long long pos_rows,
                  __nv_bfloat16* __restrict__ ypb, float* __restrict__ stats, long long M, float eps) {
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
      v[i] = *reinterpret_cast<const float4*>(z + row * C + i * 128 + lane * 4);
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
    const float* prow = pos ? pos + (row % pos_rows) * C : nullptr;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const long long off = row * C + i * 128 + lane * 4;
      const float4 o = make_float4((v[i].x - mean) * rstd * g[i].x + b[i].x, (v[i].y - mean) * rstd * g[i].y + b[i].y,
                                   (v[i].z - mean) * rstd * g[i].z + b[i].z, (v[i].w - mean) * rstd * g[i].w + b[i].w);
      if (y) *reinterpret_cast<float4*>(y + off) = o;
      if (yb) st_bf16x4(yb + off, o);
      if (ypb) {
        const float4 pv = *reinterpret_cast<const float4*>(prow + i * 128 + lane * 4);
        st_bf16x4(ypb + off, make_float4(o.x + pv.x, o.y + pv.y, o.z + pv.z, o.w + pv.w));
      }
    }
  }
}

// dz = dres + rstd*(dxhat - mean(dxhat) - xhat*mean(dxhat*xhat)), dxhat = dy*gamma, dy fp32; dgamma / dbeta as
// per-block partial rows ([gridDim.x][2][C]) folded in a fixed order by fold_partials (bit-reproducible).
template <int NCH>
__global__ void __launch_bounds__(256)
postln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ z, const float* __restrict__ gamma,
                  const float* __restrict__ stats, const float* __restrict__ dres, float* __restrict__ dz,
                  __nv_bfloat16* __restrict__ dzb, float* __restrict__ partials, long long M) {
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
    float4 xh[NCH], d[NCH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float4 xv = *reinterpret_cast<const float4*>(z + row * C + i * 128 + lane * 4);
      const float4 dv = *reinterpret_cast<const float4*>(dy + row * C + i * 128 + lane * 4);
      xh[i] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
      db[i].x += dv.x; db[i].y += dv.y; db[i].z += dv.z; db[i].w += dv.w;
      dg[i].x += dv.x * xh[i].x; dg[i].y += dv.y * xh[i].y; dg[i].z += dv.z * xh[i].z; dg[i].w += dv.w * xh[i].w;
      d[i] = make_float4(dv.x * g[i].x, dv.y * g[i].y, dv.z * g[i].z, dv.w * g[i].w);
      s1 += d[i].x + d[i].y + d[i].z + d[i].w;
      s2 += d[i].x * xh[i].x + d[i].y * xh[i].y + d[i].z * xh[i].z + d[i].w * xh[i].w;
    }
    const float c1 = warp_sum(s1) * (1.f / C), c2 = warp_sum(s2) * (1.f / C);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const long long off = row * C + i * 128 + lane * 4;
      float4 o = make_float4(rstd * (d[i].x - c1 - xh[i].x * c2), rstd * (d[i].y - c1 - xh[i].y * c2),
                             rstd * (d[i].z - c1 - xh[i].z * c2), rstd * (d[i].w - c1 - xh[i].w * c2));
      if (dres) {
        const float4 r = *reinterpret_cast<const float4*>(dres + off);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      if (dz) *reinterpret_cast<float4*>(dz + off) = o;
      if (dzb) st_bf16x4(dzb + off, o);
    }
  }
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

// xb = bf16(x); xpb = bf16(x + pos[row % pos_rows])   (4 columns per thread)
__global__ void add_pos_cast_kernel(const float* __restrict__ x, const float* __restrict__ pos, long long pos_rows,
                                    __nv_bfloat16* __restrict__ xb, __nv_bfloat16* __restrict__ xpb, long long rows, int C) {
  const int c4 = C >> 2;
  const long long total = rows * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c4;
    const int c = (int)(i % c4);
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    if (xb) st_bf16x4(xb + i * 4, v);
    if (xpb) {
      const float4 p = reinterpret_cast<const float4*>(pos)[(row % pos_rows) * c4 + c];
      st_bf16x4(xpb + i * 4, make_float4(v.x + p.x, v.y + p.y, v.z + p.z, v.w + p.w));
    }
  }
}

// ----------------------------------------------------------------------------- dropout
// out[i] = keep(i) ? in[i] / (1 - p) : 0  (+ resid[i]); keep(i) = hash(seed, i) >= p * 2^32.  The same call with
// the same seed applied to a gradient is the backward pass.  4 elements per thread.
template <bool IN_F32, bool OUT_F32>
__global__ void dropout_kernel(const void* __restrict__ in, const float* __restrict__ resid, const float* __restrict__ row_scale,
                               long long elems_per_scale, void* __restrict__ out, long long n4, uint32_t thresh, float inv_keep,
                               unsigned long long seed, const unsigned long long* __restrict__ seed_base) {
  if (seed_base) seed += *seed_base;                 // device-resident base: a captured graph sees a fresh one per replay
  const uint32_t seed_lo = (uint32_t)seed, seed_hi = (uint32_t)(seed >> 32);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v;
    if (IN_F32) {
      v = reinterpret_cast<const float4*>(in)[i];
    } else {
      const uint2 w = reinterpret_cast<const uint2*>(in)[i];
      const float2 a = unpack2(w.x), b = unpack2(w.y);
      v = make_float4(a.x, a.y, b.x, b.y);
    }
    const uint32_t hi = (uint32_t)(i >> 30), e = (uint32_t)(i << 2);   // element index = hi * 2^32 + e .. e + 3
    const float sc = row_scale ? inv_keep * row_scale[(i * 4) / elems_per_scale] : inv_keep;   // (elems_per_scale % 4 == 0)
    v.x = dropout_hash(seed_lo, seed_hi, e, hi) >= thresh ? v.x * sc : 0.f;
    v.y = dropout_hash(seed_lo, seed_hi, e + 1, hi) >= thresh ? v.y * sc : 0.f;
    v.z = dropout_hash(seed_lo, seed_hi, e + 2, hi) >= thresh ? v.z * sc : 0.f;
    v.w = dropout_hash(seed_lo, seed_hi, e + 3, hi) >= thresh ? v.w * sc : 0.f;
    if (resid) {
      const float4 r = reinterpret_cast<const float4*>(resid)[i];
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (OUT_F32) reinterpret_cast<float4*>(out)[i] = v;
    else reinterpret_cast<uint2*>(out)[i] = make_uint2(pack2(v.x, v.y), pack2(v.z, v.w));
  }
}

// ----------------------------------------------------------------------------- per-head packing
// dst[b, h, l, 0:hd] = src[(b*L + l) * ld + col0 + h*hd + :] * scale;  dst[b, h, l, hd] = extra ? extra[b*L + l] : extra_const;
// dst[b, h, l, hd+1 : DP] = 0.   One thread per 8-column piece.
__global__ void heads_pack_kernel(const __nv_bfloat16* __restrict__ src, int ld, int col0, const float* __restrict__ extra,
                                  float extra_const, __nv_bfloat16* __restrict__ dst, int B, int L, int H, int hd, int DP,
                                  float scale) {
  const int pieces = DP >> 3;
  const long long total = (long long)B * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    long long t = i / pieces;
    const int l = (int)(t % L);
    t /= L;
    const int h = (int)(t % H);
    const int b = (int)(t / H);
    const long long row = (long long)b * L + l;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (pc * 8 < hd) {
      const uint4 v = *reinterpret_cast<const uint4*>(src + row * ld + col0 + h * hd + pc * 8);
      if (scale == 1.f) {
        o = v;
      } else {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t r[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack2(w[k]);
          r[k] = pack2(f.x * scale, f.y * scale);
        }
        o = make_uint4(r[0], r[1], r[2], r[3]);
      }
    } else if (pc * 8 == hd) {
      o.x = pack2(extra ? extra[row] : extra_const, 0.f);
    }
    *reinterpret_cast<uint4*>(dst + i * 8) = o;
  }
}
// dst[(b*L + l) * ld + col0 + h*hd + :] = src[b, h, l, 0:hd] * scale
__global__ void heads_unpack_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int ld, int col0,
                                    int B, int L, int H, int hd, int DP, float scale) {
  const int pieces = hd >> 3;
  const long long total = (long long)B * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    long long t = i / pieces;
    const int l = (int)(t % L);
    t /= L;
    const int h = (int)(t % H);
    const int b = (int)(t / H);
    const uint4 v = *reinterpret_cast<const uint4*>(src + (((long long)b * H + h) * L + l) * DP + pc * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack2(w[k]);
      r[k] = pack2(f.x * scale, f.y * scale);
    }
    *reinterpret_cast<uint4*>(dst + ((long long)b * L + l) * ld + col0 + h * hd + pc * 8) = make_uint4(r[0], r[1], r[2], r[3]);
  }
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_postln_fwd(const float* z, const float* gamma, const float* beta, float eps, float* y, void* yb, const float* pos,
                     long long pos_rows, void* ypb, float* stats, long long rows, int c, void* stream) {
  if (ypb && (!pos || pos_rows <= 0)) return set_error("saicv_postln_fwd: ypb needs pos and pos_rows > 0");
  const int grid = grid_1d(rows, 8, 132 * 8);
  __nv_bfloat16* b0 = reinterpret_cast<__nv_bfloat16*>(yb);
  __nv_bfloat16* b1 = reinterpret_cast<__nv_bfloat16*>(ypb);
  switch (c) {
    case 128: postln_fwd_kernel<1><<<grid, 256, 0, ST>>>(z, gamma, beta, y, b0, pos, pos_rows, b1, stats, rows, eps); break;
    case 256: postln_fwd_kernel<2><<<grid, 256, 0, ST>>>(z, gamma, beta, y, b0, pos, pos_rows, b1, stats, rows, eps); break;
    case 384: postln_fwd_kernel<3><<<grid, 256, 0, ST>>>(z, gamma, beta, y, b0, pos, pos_rows, b1, stats, rows, eps); break;
    case 512: postln_fwd_kernel<4><<<grid, 256, 0, ST>>>(z, gamma, beta, y, b0, pos, pos_rows, b1, stats, rows, eps); break;
    default: return set_error("saicv_postln_fwd: unsupported width %d", c);
  }
  return check_launch("postln_fwd_kernel");
}

int saicv_postln_bwd(const float* dy, const float* z, const float* gamma, const float* stats, const float* dres, float* dz,
                     void* dzb, float* partials, float* dgamma, float* dbeta, long long rows, int c, int accumulate,
                     void* stream) {
  if (!partials) return set_error("saicv_postln_bwd: needs a [SAICV_BN_PARTIAL_ROWS][2*c] fp32 workspace");
  const int grid = grid_1d(rows, 8 * 8, 132 * 2);
  __nv_bfloat16* b0 = reinterpret_cast<__nv_bfloat16*>(dzb);
  switch (c) {
    case 128: postln_bwd_kernel<1><<<grid, 256, 0, ST>>>(dy, z, gamma, stats, dres, dz, b0, partials, rows); break;
    case 256: postln_bwd_kernel<2><<<grid, 256, 0, ST>>>(dy, z, gamma, stats, dres, dz, b0, partials, rows); break;
    case 384: postln_bwd_kernel<3><<<grid, 256, 0, ST>>>(dy, z, gamma, stats, dres, dz, b0, partials, rows); break;
    case 512: postln_bwd_kernel<4><<<grid, 256, 0, ST>>>(dy, z, gamma, stats, dres, dz, b0, partials, rows); break;
    default: return set_error("saicv_postln_bwd: unsupported width %d", c);
  }
  if (int e = check_launch("postln_bwd_kernel")) return e;
  return fold_partials(partials, grid, 2 * c, dgamma, dbeta, c, accumulate, ST);
}

int saicv_add_pos_cast(const float* x, const float* pos, long long pos_rows, void* xb, void* xpb, long long rows, int c,
                       void* stream) {
  if (c % 4) return set_error("saicv_add_pos_cast: C %% 4 != 0");
  if (xpb && (!pos || pos_rows <= 0)) return set_error("saicv_add_pos_cast: xpb needs pos and pos_rows > 0");
  add_pos_cast_kernel<<<grid_1d(rows * (c / 4)), 256, 0, ST>>>(x, pos, pos_rows, reinterpret_cast<__nv_bfloat16*>(xb),
                                                               reinterpret_cast<__nv_bfloat16*>(xpb), rows, c);
  return check_launch("add_pos_cast_kernel");
}

int saicv_dropout(const void* in, int in_f32, const float* resid, const float* row_scale, long long elems_per_scale, void* out,
                  int out_f32, long long n, float p, unsigned long long seed, const unsigned long long* seed_base, void* stream) {
  if (row_scale && (elems_per_scale <= 0 || elems_per_scale % 4)) return set_error("saicv_dropout: elems_per_scale must be a positive multiple of 4");
  if (n % 4) return set_error("saicv_dropout: n %% 4 != 0");
  if (!(p >= 0.f && p < 1.f)) return set_error("saicv_dropout: p must be in [0, 1)");
  if (resid && !out_f32) return set_error("saicv_dropout: a residual needs an fp32 output");
  const uint32_t thresh = dropout_threshold(p);
  const float inv_keep = 1.f / (1.f - p);
  const int grid = grid_1d(n / 4);
  if (in_f32 && out_f32) dropout_kernel<true, true><<<grid, 256, 0, ST>>>(in, resid, row_scale, elems_per_scale, out, n / 4, thresh, inv_keep, seed, seed_base);
  else if (in_f32) dropout_kernel<true, false><<<grid, 256, 0, ST>>>(in, resid, row_scale, elems_per_scale, out, n / 4, thresh, inv_keep, seed, seed_base);
  else if (out_f32) dropout_kernel<false, true><<<grid, 256, 0, ST>>>(in, resid, row_scale, elems_per_scale, out, n / 4, thresh, inv_keep, seed, seed_base);
  else dropout_kernel<false, false><<<grid, 256, 0, ST>>>(in, resid, row_scale, elems_per_scale, out, n / 4, thresh, inv_keep, seed, seed_base);
  return check_launch("dropout_kernel");
}

int saicv_heads_pack(const void* src, int ld, int col0, const float* extra, float extra_const, void* dst, int b, int l, int h,
                     int hd, int dp, float scale, void* stream) {
  if (hd % 8 || dp % 8 || dp <= hd || ld % 8 || col0 % 8) return set_error("saicv_heads_pack: hd, dp, ld, col0 must be multiples of 8 and dp > hd");
  heads_pack_kernel<<<grid_1d((long long)b * h * l * (dp / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), ld, col0, extra, extra_const, reinterpret_cast<__nv_bfloat16*>(dst), b, l, h, hd, dp, scale);
  return check_launch("heads_pack_kernel");
}

int saicv_heads_unpack(const void* src, void* dst, int ld, int col0, int b, int l, int h, int hd, int dp, float scale,
                       void* stream) {
  if (hd % 8 || dp % 8 || ld % 8 || col0 % 8) return set_error("saicv_heads_unpack: hd, dp, ld, col0 must be multiples of 8");
  heads_unpack_kernel<<<grid_1d((long long)b * h * l * (hd / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<__nv_bfloat16*>(dst), ld, col0, b, l, h, hd, dp, scale);
  return check_launch("heads_unpack_kernel");
}

}  // extern "C"
