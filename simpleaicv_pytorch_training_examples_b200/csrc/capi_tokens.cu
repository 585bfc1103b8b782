// Token gather / scatter for masked-token models (SURVEY.md 8 f4: MAE pre-training,
// SimpleAICV/masked_image_modeling/models/vit_mae.py): one kernel pair serves both places where the reference shuffles
// tokens with torch.gather on an index repeated over the channel axis, concatenates a learned token and adds the
// position encoding:
//   encoder (:171-186)  keep the un-masked patch tokens:   out[b, 0] = cls_token + pos[0],  out[b, 1+i] = x[b, keep[b, i]] + pos[1 + keep[b, i]]
//   decoder (:339-354)  un-shuffle and fill mask tokens:   out[b, 0] = y[b, 0] + pos[0],    out[b, 1+j] = (r < Lk ? y[b, 1+r] : mask_token) + pos[1+j],  r = restore[b, j]
// Generic form:  out[b, r, :] = (idx[b, r] >= 0 ? src[b, idx[b, r], :] : fill[:]) + pos[pos_idx ? pos_idx[b, r] : r, :]
// The backward scatters dout rows back to the source rows they came from (every source row is referenced at most once;
// unreferenced rows are zero) and sums the rows that took `fill` (per-slab partials, folded in a fixed order).
// fp32 residual-stream tensors, HBM-bound, 16-byte vectors.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"

namespace saicv {
namespace {

constexpr int kTokThreads = 256;

__global__ void __launch_bounds__(kTokThreads)
token_gather_fwd_kernel(const float4* __restrict__ src, long long src_rows, const int* __restrict__ idx, const float4* __restrict__ fill,
                        const float4* __restrict__ pos, const int* __restrict__ pos_idx, float4* __restrict__ out, long long rows_total,
                        int R, int c4) {
  const long long total = rows_total * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c4;
    const int v = (int)(i - row * c4);
    const long long b = row / R;
    const int r = (int)(row - b * R);
    const int s = __ldg(idx + row);
    float4 a = s >= 0 ? __ldg(src + (b * src_rows + s) * c4 + v) : __ldg(fill + v);
    if (pos != nullptr) {
      const int pr = pos_idx != nullptr ? __ldg(pos_idx + row) : r;
      const float4 p = __ldg(pos + (long long)pr * c4 + v);
      a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
    }
    out[i] = a;
  }
}

// dsrc (fp32 or bf16, pre-zeroed by the caller when some source rows are unreferenced) <- dout rows with idx >= 0
template <bool BF16>
__global__ void __launch_bounds__(kTokThreads)
token_gather_bwd_kernel(const float4* __restrict__ dout, const int* __restrict__ idx, void* __restrict__ dsrc, long long src_rows,
                        long long rows_total, int R, int c4) {
  const long long total = rows_total * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c4;
    const int v = (int)(i - row * c4);
    const int s = __ldg(idx + row);
    if (s < 0) continue;
    const long long b = row / R;
    const float4 g = __ldg(dout + i);
    const long long o = (b * src_rows + s) * c4 + v;
    if (BF16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(g.x, g.y), hi = __floats2bfloat162_rn(g.z, g.w);
      reinterpret_cast<uint2*>(dsrc)[o] = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
    } else {
      reinterpret_cast<float4*>(dsrc)[o] = g;
    }
  }
}

// partial[slab][c] = sum over the rows of the slab with idx < 0 of dout[row][c]; grid (C / 32, nslab), block (32, 8)
__global__ void __launch_bounds__(256)
token_fill_grad_kernel(const float* __restrict__ dout, const int* __restrict__ idx, float* __restrict__ partial, long long rows_total,
                       int C, long long rows_per_slab) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * rows_per_slab;
  long long r1 = r0 + rows_per_slab;
  if (r1 > rows_total) r1 = rows_total;
  float s = 0.f;
  if (col < C)
    for (long long r = r0 + threadIdx.y; r < r1; r += 8)
      if (__ldg(idx + r) < 0) s += __ldg(dout + r * C + col);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    partial[(long long)blockIdx.y * C + col] = t;
  }
}

int blocks_for(long long items) {
  long long b = (items + kTokThreads - 1) / kTokThreads;
  return (int)(b < 1 ? 1 : b > 132 * 16 ? 132 * 16 : b);
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST reinterpret_cast<cudaStream_t>(stream)

extern "C" {

int saicv_token_gather_fwd(const float* src, long long src_rows, const int* idx, const float* fill, const float* pos,
                           const int* pos_idx, float* out, int b, int r, int c, void* stream) {
  if (c % 4) return set_error("saicv_token_gather_fwd: C %% 4 != 0");
  const long long rows = (long long)b * r;
  token_gather_fwd_kernel<<<blocks_for(rows * (c / 4)), kTokThreads, 0, ST>>>(
      reinterpret_cast<const float4*>(src), src_rows, idx, reinterpret_cast<const float4*>(fill), reinterpret_cast<const float4*>(pos),
      pos_idx, reinterpret_cast<float4*>(out), rows, r, c / 4);
  return check_launch("token_gather_fwd_kernel");
}

int saicv_token_fill_slabs(long long rows) {
  const long long s = (rows + 511) / 512;
  return (int)(s < 1 ? 1 : s > 128 ? 128 : s);
}

int saicv_token_gather_bwd(const float* dout, const int* idx, void* dsrc, int dsrc_bf16, long long src_rows,
                           float* fill_partial, int b, int r, int c, void* stream) {
  if (c % 4) return set_error("saicv_token_gather_bwd: C %% 4 != 0");
  const long long rows = (long long)b * r;
  if (dsrc != nullptr) {
    if (dsrc_bf16)
      token_gather_bwd_kernel<true><<<blocks_for(rows * (c / 4)), kTokThreads, 0, ST>>>(reinterpret_cast<const float4*>(dout), idx, dsrc,
                                                                                         src_rows, rows, r, c / 4);
    else
      token_gather_bwd_kernel<false><<<blocks_for(rows * (c / 4)), kTokThreads, 0, ST>>>(reinterpret_cast<const float4*>(dout), idx, dsrc,
                                                                                          src_rows, rows, r, c / 4);
    if (check_launch("token_gather_bwd_kernel")) return 1;
  }
  if (fill_partial != nullptr) {
    const int nslab = saicv_token_fill_slabs(rows);
    const long long per = (rows + nslab - 1) / nslab;
    token_fill_grad_kernel<<<dim3((c + 31) / 32, nslab), dim3(32, 8), 0, ST>>>(dout, idx, fill_partial, rows, c, per);
    if (check_launch("token_fill_grad_kernel")) return 1;
  }
  return 0;
}

}  // extern "C"
