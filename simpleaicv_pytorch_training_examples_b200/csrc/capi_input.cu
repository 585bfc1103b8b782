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

}  // namespace
}  // namespace saicv

using namespace saicv;

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
    const int blocks = (int)((groups + kInThreads - 1) / kInThreads < 132 * 16 ? (groups + kInThreads - 1) / kInThreads : 132 * 16);
    u8_nhwc_to_nchw_norm_vec_kernel<<<blocks, kInThreads, 0, st>>>(reinterpret_cast<const uint32_t*>(in), out, groups, (int)(hw / 4), nm);
    return check_launch("u8_nhwc_to_nchw_norm_vec_kernel");
  }
  const int blocks = (int)((pixels + kInThreads - 1) / kInThreads < 132 * 16 ? (pixels + kInThreads - 1) / kInThreads : 132 * 16);
  u8_nhwc_to_nchw_norm_kernel<<<blocks, kInThreads, 0, st>>>(reinterpret_cast<const uint8_t*>(in), out, pixels, hw, nm);
  return check_launch("u8_nhwc_to_nchw_norm_kernel");
}
