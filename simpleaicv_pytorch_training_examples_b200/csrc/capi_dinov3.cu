// DINOv3 ViT kernels (SimpleAICV/detection/models/backbones/dinov3vit.py): rotary position embedding applied in place to
// the q and k slices of the packed qkv GEMM output (:271-282 rope_rotate_half / rope_apply, :347-367 apply_rope) and its
// transpose on dq / dk, and the SwiGLU gate of the *_plus variants (:117-141).
//
// Rounding points are the reference's under autocast: apply_rope casts q and k to the fp32 table's dtype, computes
// x*cos + rotate_half(x)*sin as two separately rounded products and one add, then rounds to bf16.  __fmul_rn /
// __fadd_rn keep nvcc from contracting that into an FMA, so the result is bit-identical to the torch expression.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"
#include "vec8.cuh"

namespace saicv {
namespace {

__device__ __forceinline__ void load4(const __nv_bfloat16* p, float (&f)[4]) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  f[0] = __uint_as_float(v.x << 16);
  f[1] = __uint_as_float(v.x & 0xffff0000u);
  f[2] = __uint_as_float(v.y << 16);
  f[3] = __uint_as_float(v.y & 0xffff0000u);
}
__device__ __forceinline__ void store4(__nv_bfloat16* p, const float (&f)[4]) {
  __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
  *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&b));
}

// One thread = 4 columns j..j+3 of the first half of one (row, q|k, head) vector and their partners j+half..j+half+3.
//   forward:  y[j] = x[j] cos[j] + (-x[j+h]) sin[j];        y[j+h] = x[j+h] cos[j+h] + x[j] sin[j+h]
//   backward: dx[j] = g[j] cos[j] + g[j+h] sin[j+h];        dx[j+h] = g[j+h] cos[j+h] - g[j] sin[j]
template <bool BWD>
__global__ void __launch_bounds__(256) rope_qk_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ sin_t,
                                                      const float* __restrict__ cos_t, long long rows, int L, int heads, int hd) {
  const int half = hd >> 1, q4 = half >> 2;
  const long long total = rows * 2 * heads * q4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % q4);
    const long long vec = i / q4;                 // (row, slot, head) with slot in {q, k}
    const int head = (int)(vec % heads);
    const int slot = (int)((vec / heads) % 2);
    const long long row = vec / (2LL * heads);
    const int l = (int)(row % L);
    const int j = c * 4;
    __nv_bfloat16* p = qkv + ((row * 3 + slot) * heads + head) * (long long)hd;
    const float* sn = sin_t + (long long)l * hd;
    const float* cs = cos_t + (long long)l * hd;
    const float4 s0 = *reinterpret_cast<const float4*>(sn + j), s1 = *reinterpret_cast<const float4*>(sn + j + half);
    const float4 c0 = *reinterpret_cast<const float4*>(cs + j), c1 = *reinterpret_cast<const float4*>(cs + j + half);
    const float sa[4] = {s0.x, s0.y, s0.z, s0.w}, sb[4] = {s1.x, s1.y, s1.z, s1.w};
    const float ca[4] = {c0.x, c0.y, c0.z, c0.w}, cb[4] = {c1.x, c1.y, c1.z, c1.w};
    float a[4], b[4], ya[4], yb[4];
    load4(p + j, a);
    load4(p + j + half, b);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (BWD) {
        ya[k] = __fadd_rn(__fmul_rn(a[k], ca[k]), __fmul_rn(b[k], sb[k]));
        yb[k] = __fadd_rn(__fmul_rn(b[k], cb[k]), -__fmul_rn(a[k], sa[k]));
      } else {
        ya[k] = __fadd_rn(__fmul_rn(a[k], ca[k]), __fmul_rn(-b[k], sa[k]));
        yb[k] = __fadd_rn(__fmul_rn(b[k], cb[k]), __fmul_rn(a[k], sb[k]));
      }
    }
    store4(p + j, ya);
    store4(p + j + half, yb);
  }
}

// F.silu of a bf16 tensor: computed in fp32 as x / (1 + exp(-x)) and rounded to bf16 (torch's silu kernel).
__device__ __forceinline__ float silu_bf16(float x) {
  return __bfloat162float(__float2bfloat16_rn(__fdiv_rn(x, __fadd_rn(1.f, expf(-x)))));
}

// h = bf16(silu(a)) * b, rounded to bf16
__global__ void swiglu_fwd_kernel(const V8* __restrict__ a, const V8* __restrict__ b, V8* __restrict__ h, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(ldg8(a, i), x);
    unpack8(ldg8(b, i), y);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = __fmul_rn(silu_bf16(x[k]), y[k]);
    stg8(h, i, pack8(x));
  }
}

// db = bf16(dh * bf16(silu(a)));  ds = bf16(dh * b);  da = bf16(ds * sig(a) * (1 + a (1 - sig(a))))   (autograd's order)
__global__ void swiglu_bwd_kernel(const V8* __restrict__ dh, const V8* __restrict__ a, const V8* __restrict__ b,
                                  V8* __restrict__ da, V8* __restrict__ db, long long nvec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[8], x[8], y[8], ga[8], gb[8];
    unpack8(ldg8(dh, i), g);
    unpack8(ldg8(a, i), x);
    unpack8(ldg8(b, i), y);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      gb[k] = __fmul_rn(g[k], silu_bf16(x[k]));
      const float ds = __bfloat162float(__float2bfloat16_rn(__fmul_rn(g[k], y[k])));
      const float sg = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x[k])));
      ga[k] = __fmul_rn(__fmul_rn(ds, sg), __fadd_rn(1.f, __fmul_rn(x[k], __fsub_rn(1.f, sg))));
    }
    stg8(da, i, pack8(ga));
    stg8(db, i, pack8(gb));
  }
}

int rope_launch(bool bwd, void* qkv, const float* sin_t, const float* cos_t, int b, int l, int heads, int hd, void* stream) {
  const char* name = bwd ? "saicv_rope_qk_bwd" : "saicv_rope_qk_fwd";
  if (hd <= 0 || hd % 8) return set_error("%s: head size %d must be a positive multiple of 8", name, hd);
  if (b <= 0 || l <= 0 || heads <= 0) return set_error("%s: empty shape (b %d, L %d, heads %d)", name, b, l, heads);
  if (!qkv || !sin_t || !cos_t) return set_error("%s: NULL pointer", name);
  const long long rows = (long long)b * l;
  const long long items = rows * 2 * heads * (hd / 8);
  __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(qkv);
  cudaStream_t st = (cudaStream_t)stream;
  if (bwd) rope_qk_kernel<true><<<grid_1d(items), 256, 0, st>>>(p, sin_t, cos_t, rows, l, heads, hd);
  else rope_qk_kernel<false><<<grid_1d(items), 256, 0, st>>>(p, sin_t, cos_t, rows, l, heads, hd);
  return check_launch(bwd ? "rope_qk_kernel<bwd>" : "rope_qk_kernel<fwd>");
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST ((cudaStream_t)stream)

extern "C" {

int saicv_rope_qk_fwd(void* qkv, const float* sin_t, const float* cos_t, int b, int l, int heads, int hd, void* stream) {
  return rope_launch(false, qkv, sin_t, cos_t, b, l, heads, hd, stream);
}

int saicv_rope_qk_bwd(void* dqkv, const float* sin_t, const float* cos_t, int b, int l, int heads, int hd, void* stream) {
  return rope_launch(true, dqkv, sin_t, cos_t, b, l, heads, hd, stream);
}

int saicv_swiglu_fwd(const void* a, const void* b, void* h, long long n, void* stream) {
  if (n % 8) return set_error("saicv_swiglu_fwd: n %% 8 != 0");
  swiglu_fwd_kernel<<<grid_1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const V8*>(a), reinterpret_cast<const V8*>(b),
                                                    reinterpret_cast<V8*>(h), n / 8);
  return check_launch("swiglu_fwd_kernel");
}

int saicv_swiglu_bwd(const void* dh, const void* a, const void* b, void* da, void* db, long long n, void* stream) {
  if (n % 8) return set_error("saicv_swiglu_bwd: n %% 8 != 0");
  swiglu_bwd_kernel<<<grid_1d(n / 8), 256, 0, ST>>>(reinterpret_cast<const V8*>(dh), reinterpret_cast<const V8*>(a),
                                                    reinterpret_cast<const V8*>(b), reinterpret_cast<V8*>(da),
                                                    reinterpret_cast<V8*>(db), n / 8);
  return check_launch("swiglu_bwd_kernel");
}

}  // extern "C"
