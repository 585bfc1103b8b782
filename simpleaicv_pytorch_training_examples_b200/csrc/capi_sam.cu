// SAM image-encoder specific kernels (SimpleAICV/interactive_segmentation/models/segment_anything/image_encoder.py):
//   window partition / unpartition with zero padding (:32-79),
//   decomposed relative-position bias (:82-144): the bias rel_h[q, kh] + rel_w[q, kw] is turned into extra score
//   columns so that the wgmma attention kernel adds it on the tensor cores:
//       Qe[l] = [ q[l] * scale | rel_h[l, 0..Sh) | rel_w[l, 0..Sw) | 0 ]      rel_h[l, kh] = q[l] . Rh[qh(l) - kh + Sh - 1]
//       Ke[l] = [ k[l]         | onehot(kh(l))   | onehot(kw(l))   | 0 ]
//       Qe . Ke^T = scale * q.k + rel_h[q, kh(k)] + rel_w[q, kw(k)]            (= image_encoder.py:171-174)
//   and the matching backward (dq from dQe, d rel_pos_h / d rel_pos_w with a fixed-order two-stage reduction),
//   the positional-embedding broadcast add (:315).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"
#include "vec8.cuh"

namespace saicv {
namespace {

// windows[(b*nwy+wy)*nwx+wx][iy*ws+ix][c] = x[b][wy*ws+iy][wx*ws+ix][c]  (0 outside H x W)
__global__ void window_partition_kernel(const V8* __restrict__ x, V8* __restrict__ win, int B, int H, int W, int C, int ws, int nwy,
                                        int nwx) {
  const int vpr = C >> 3;
  const long long total = (long long)B * nwy * nwx * ws * ws * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int ix = (int)(t % ws); t /= ws;
    const int iy = (int)(t % ws); t /= ws;
    const int wx = (int)(t % nwx); t /= nwx;
    const int wy = (int)(t % nwy);
    const long long b = t / nwy;
    const int h = wy * ws + iy, w = wx * ws + ix;
    V8 val;
    val.zero();
    if (h < H && w < W) val = x[((b * H + h) * W + w) * vpr + v];
    win[i] = val;
  }
}
// x[b][h][w][c] = windows[...] (padding rows dropped)
__global__ void window_unpartition_kernel(const V8* __restrict__ win, V8* __restrict__ x, int B, int H, int W, int C, int ws,
                                          int nwy, int nwx) {
  const int vpr = C >> 3;
  const long long total = (long long)B * H * W * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H);
    const long long b = t / H;
    const int wy = h / ws, iy = h % ws, wx = w / ws, ix = w % ws;
    x[i] = win[((((b * nwy + wy) * nwx + wx) * ws + iy) * ws + ix) * vpr + v];
  }
}

// x[b][r][c] += pos[r][c]   (fp32, in place)
__global__ void add_pos_kernel(float4* __restrict__ x, const float4* __restrict__ pos, long long per_batch4, long long total4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = x[i];
    const float4 p = pos[i % per_batch4];
    a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
    x[i] = a;
  }
}

// ---- rel-pos score columns.  qkv: [Bw][L][3][H][hd] bf16 (L = Sh*Sw tokens, row-major (qh, qw)); rows r of the
// per-head operands are ordered (window, head, token).  The bias terms are dot products of q rows with rel-pos table
// rows, i.e. GEMMs; the kernels here only move / re-index data around three launches of the tensor-core engine:
//   forward   T[r][idx] = q[r] . Rtab[idx]                      (saicv_linear_fwd:  qc [rows, hd] x rtab [nip, hd]^T)
//             Qe[r] = [q[r] * scale | T[r][qh - kh + Sh - 1], kh < Sh | T[r][nh + qw - kw + Sw - 1], kw < Sw | 0]
//   backward  ef[r][idx] = the bias-column gradients re-indexed so that column idx is the table row it belongs to
//             dq[r]  = scale * dQe[r][0:hd] + ef[r] . Rtab        (saicv_linear_dgrad: ef [rows, nip] x rtab [nip, hd])
//             dRtab  = ef^T . qc                                  (saicv_linear_wgrad)
// Rtab = [rel_pos_h ; rel_pos_w ; 0] as bf16 [nip][hd] (the reference's einsum consumes the tables in bf16 under autocast).

// qc[r][0:hd] = q row of (window, head, token) r, unscaled; one thread per 16-byte piece
__global__ void relpos_packq_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ qc, int Bw, int H, int L, int hd) {
  const int pieces = hd >> 3;
  const long long total = (long long)Bw * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    const long long r = i / pieces;
    const int l = (int)(r % L);
    const long long bh = r / L;
    const int h = (int)(bh % H);
    const long long bw = bh / H;
    reinterpret_cast<uint4*>(qc)[i] =
        __ldg(reinterpret_cast<const uint4*>(qkv + ((bw * L + l) * 3) * (long long)H * hd + (long long)h * hd + pc * 8));
  }
}

// rtab[idx][c] = bf16(rel_pos_h[idx][c]) for idx < nh, bf16(rel_pos_w[idx - nh][c]) for idx < nh + nw, else 0
__global__ void relpos_table_kernel(const float* __restrict__ rph, const float* __restrict__ rpw, __nv_bfloat16* __restrict__ rtab,
                                    int nh, int nw, int nip, int hd) {
  const int total = nip * hd;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int idx = i / hd, c = i % hd;
    const float v = idx < nh ? rph[idx * hd + c] : (idx < nh + nw ? rpw[(idx - nh) * hd + c] : 0.f);
    rtab[i] = __float2bfloat16_rn(v);
  }
}

// Qe / Ke rows from qkv and T; one thread per 16-byte piece of a Qe row and the matching piece of the Ke row
__global__ void __launch_bounds__(256)
relpos_gather_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ T, __nv_bfloat16* __restrict__ qe,
                     __nv_bfloat16* __restrict__ ke, int Bw, int H, int Sh, int Sw, int hd, int DQK, int NIP, float scale) {
  const int L = Sh * Sw, pieces = DQK >> 3, nh = 2 * Sh - 1;
  const long long total = (long long)Bw * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    const long long r = i / pieces;
    const int l = (int)(r % L);
    const long long bh = r / L;
    const int h = (int)(bh % H);
    const long long bw = bh / H;
    const int qh = l / Sw, qw = l % Sw;
    uint4 qo = make_uint4(0u, 0u, 0u, 0u), ko = make_uint4(0u, 0u, 0u, 0u);
    if (pc * 8 < hd) {
      const __nv_bfloat16* qrow = qkv + ((bw * L + l) * 3) * (long long)H * hd + (long long)h * hd + pc * 8;
      const uint4 qv = __ldg(reinterpret_cast<const uint4*>(qrow));
      ko = __ldg(reinterpret_cast<const uint4*>(qrow + (long long)H * hd));
      const uint32_t w[4] = {qv.x, qv.y, qv.z, qv.w};
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        __nv_bfloat162 v = __floats2bfloat162_rn(__uint_as_float(w[k] << 16) * scale, __uint_as_float(w[k] & 0xffff0000u) * scale);
        o[k] = *reinterpret_cast<uint32_t*>(&v);
      }
      qo = make_uint4(o[0], o[1], o[2], o[3]);
    } else {
      const unsigned short* trow = reinterpret_cast<const unsigned short*>(T + r * NIP);
      uint32_t qw4[4], kw4[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        unsigned short qv[2], kv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = pc * 8 + 2 * k + e - hd;           // bias column: key row j (< Sh) or key column j - Sh
          qv[e] = 0;
          kv[e] = 0;
          if (j < Sh) {
            qv[e] = __ldg(trow + (qh - j + Sh - 1));
            kv[e] = j == qh ? (unsigned short)0x3F80 : (unsigned short)0;     // bf16 1.0
          } else if (j < Sh + Sw) {
            qv[e] = __ldg(trow + nh + (qw - (j - Sh) + Sw - 1));
            kv[e] = (j - Sh) == qw ? (unsigned short)0x3F80 : (unsigned short)0;
          }
        }
        qw4[k] = (uint32_t)qv[0] | ((uint32_t)qv[1] << 16);
        kw4[k] = (uint32_t)kv[0] | ((uint32_t)kv[1] << 16);
      }
      qo = make_uint4(qw4[0], qw4[1], qw4[2], qw4[3]);
      ko = make_uint4(kw4[0], kw4[1], kw4[2], kw4[3]);
    }
    reinterpret_cast<uint4*>(qe)[i] = qo;
    reinterpret_cast<uint4*>(ke)[i] = ko;
  }
}

// dqkv q slot of row r = bf16(scale * dQe[r][0:hd] + dqx[r][0:hd]); dqx fp32 (the table term from the dgrad GEMM)
__global__ void relpos_dq_combine_kernel(const __nv_bfloat16* __restrict__ dqe, const float* __restrict__ dqx, __nv_bfloat16* __restrict__ dqkv,
                                         int Bw, int H, int L, int hd, int DQK, float scale) {
  const int pieces = hd >> 3;
  const long long total = (long long)Bw * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    const long long r = i / pieces;
    const int l = (int)(r % L);
    const long long bh = r / L;
    const int h = (int)(bh % H);
    const long long bw = bh / H;
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(dqe + r * DQK + pc * 8));
    const float4 x0 = __ldg(reinterpret_cast<const float4*>(dqx + r * hd + pc * 8));
    const float4 x1 = __ldg(reinterpret_cast<const float4*>(dqx + r * hd + pc * 8 + 4));
    const uint32_t w[4] = {g.x, g.y, g.z, g.w};
    const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      __nv_bfloat162 v = __floats2bfloat162_rn(fmaf(__uint_as_float(w[k] << 16), scale, xs[2 * k]),
                                               fmaf(__uint_as_float(w[k] & 0xffff0000u), scale, xs[2 * k + 1]));
      o[k] = *reinterpret_cast<uint32_t*>(&v);
    }
    *reinterpret_cast<uint4*>(dqkv + ((bw * L + l) * 3) * (long long)H * hd + (long long)h * hd + pc * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ef[r][idx] = dT_h[r][qh(r) - idx + Sh - 1] (idx < nh), ef[r][nh + idx] = dT_w[r][qw(r) - idx + Sw - 1] (idx < nw), zero where
// the key index falls outside the grid and in the padding columns up to NIP; dT = the bias columns of dQe.
__global__ void __launch_bounds__(256)
relpos_shift_kernel(const __nv_bfloat16* __restrict__ dqe, __nv_bfloat16* __restrict__ ef, int Bw, int H, int Sh, int Sw, int hd,
                    int DQK, int NIP) {
  const int L = Sh * Sw;
  const int pieces = NIP >> 3;
  const int nh = 2 * Sh - 1, nw = 2 * Sw - 1;
  const long long total = (long long)Bw * H * L * pieces;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pc = (int)(i % pieces);
    const long long r = i / pieces;
    const int l = (int)(r % L);
    const int qh = l / Sw, qw = l % Sw;
    const unsigned short* gs = reinterpret_cast<const unsigned short*>(dqe + r * DQK + hd);
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      unsigned short v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int idx = pc * 8 + 2 * k + e;
        int src = -1;
        if (idx < nh) {
          const int kh = qh - idx + Sh - 1;
          if (kh >= 0 && kh < Sh) src = kh;
        } else if (idx < nh + nw) {
          const int kw = qw - (idx - nh) + Sw - 1;
          if (kw >= 0 && kw < Sw) src = Sh + kw;
        }
        v[e] = src >= 0 ? __ldg(gs + src) : (unsigned short)0;
      }
      w[k] = (uint32_t)v[0] | ((uint32_t)v[1] << 16);
    }
    reinterpret_cast<uint4*>(ef)[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_window_partition(const void* x, void* windows, int b, int h, int w, int c, int ws, void* stream) {
  if (c % 8 || ws < 1) return set_error("saicv_window_partition: C %% 8 != 0 or bad window size");
  const int nwy = (h + ws - 1) / ws, nwx = (w + ws - 1) / ws;
  window_partition_kernel<<<grid_1d((long long)b * nwy * nwx * ws * ws * (c / 8)), 256, 0, ST>>>(
      reinterpret_cast<const V8*>(x), reinterpret_cast<V8*>(windows), b, h, w, c, ws, nwy, nwx);
  return check_launch("window_partition_kernel");
}

int saicv_window_unpartition(const void* windows, void* x, int b, int h, int w, int c, int ws, void* stream) {
  if (c % 8 || ws < 1) return set_error("saicv_window_unpartition: C %% 8 != 0 or bad window size");
  const int nwy = (h + ws - 1) / ws, nwx = (w + ws - 1) / ws;
  window_unpartition_kernel<<<grid_1d((long long)b * h * w * (c / 8)), 256, 0, ST>>>(
      reinterpret_cast<const V8*>(windows), reinterpret_cast<V8*>(x), b, h, w, c, ws, nwy, nwx);
  return check_launch("window_unpartition_kernel");
}

int saicv_add_pos_embed(float* x, const float* pos, int b, long long per_batch, void* stream) {
  if (per_batch % 4) return set_error("saicv_add_pos_embed: per-batch size %% 4 != 0");
  add_pos_kernel<<<grid_1d((long long)b * per_batch / 4), 256, 0, ST>>>(reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(pos),
                                                                      per_batch / 4, (long long)b * per_batch / 4);
  return check_launch("add_pos_kernel");
}

static int relpos_check(const char* who, int hd, int sh, int sw, int dqk, int nip) {
  if (hd % 8 || dqk % 8 || dqk < hd + sh + sw) return set_error("%s: dqk %d too small for %d + %d + %d (or not a multiple of 8)", who, dqk, hd, sh, sw);
  if (nip % 8 || nip < 2 * sh - 1 + 2 * sw - 1) return set_error("%s: nip must be a multiple of 8 covering both tables", who);
  return 0;
}

int saicv_relpos_pack_q(const void* qkv, void* qc, int bw, int heads, int hd, int l, void* stream) {
  if (hd % 8) return set_error("saicv_relpos_pack_q: hd %% 8 != 0");
  relpos_packq_kernel<<<grid_1d((long long)bw * heads * l * (hd / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(qc), bw, heads, l, hd);
  return check_launch("relpos_packq_kernel");
}

int saicv_relpos_table(const float* rel_pos_h, const float* rel_pos_w, void* rtab, int sh, int sw, int nip, int hd, void* stream) {
  if (nip < 2 * sh - 1 + 2 * sw - 1) return set_error("saicv_relpos_table: nip too small");
  relpos_table_kernel<<<grid_1d((long long)nip * hd), 256, 0, ST>>>(rel_pos_h, rel_pos_w, reinterpret_cast<__nv_bfloat16*>(rtab), 2 * sh - 1,
                                                                 2 * sw - 1, nip, hd);
  return check_launch("relpos_table_kernel");
}

int saicv_relpos_gather(const void* qkv, const void* t, void* qe, void* ke, int bw, int heads, int hd, int sh, int sw, int dqk, int nip,
                        float scale, void* stream) {
  if (int e = relpos_check("saicv_relpos_gather", hd, sh, sw, dqk, nip)) return e;
  relpos_gather_kernel<<<grid_1d((long long)bw * heads * sh * sw * (dqk / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<const __nv_bfloat16*>(t), reinterpret_cast<__nv_bfloat16*>(qe),
      reinterpret_cast<__nv_bfloat16*>(ke), bw, heads, sh, sw, hd, dqk, nip, scale);
  return check_launch("relpos_gather_kernel");
}

int saicv_relpos_shift(const void* dqe, void* ef, int bw, int heads, int hd, int sh, int sw, int dqk, int nip, void* stream) {
  if (int e = relpos_check("saicv_relpos_shift", hd, sh, sw, dqk, nip)) return e;
  relpos_shift_kernel<<<grid_1d((long long)bw * heads * sh * sw * (nip / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(dqe), reinterpret_cast<__nv_bfloat16*>(ef), bw, heads, sh, sw, hd, dqk, nip);
  return check_launch("relpos_shift_kernel");
}

int saicv_relpos_dq_combine(const void* dqe, const float* dqx, void* dqkv, int bw, int heads, int hd, int l, int dqk, float scale,
                            void* stream) {
  if (hd % 8 || dqk % 8) return set_error("saicv_relpos_dq_combine: hd, dqk must be multiples of 8");
  relpos_dq_combine_kernel<<<grid_1d((long long)bw * heads * l * (hd / 8)), 256, 0, ST>>>(
      reinterpret_cast<const __nv_bfloat16*>(dqe), dqx, reinterpret_cast<__nv_bfloat16*>(dqkv), bw, heads, l, hd, dqk, scale);
  return check_launch("relpos_dq_combine_kernel");
}

}  // extern "C"
