// Eight bf16 values as ONE 16-byte vector.  The storage is a uint4 so that every global access is a single
// LDG.128 / STG.128: a struct of four __nv_bfloat162 members is split by the compiler into four 32-bit accesses,
// which quadruples the L1 wavefronts of the streaming kernels.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>

namespace saicv {

struct V8 {
  uint4 q;
  __device__ __forceinline__ __nv_bfloat162 h(int k) const {
    const uint32_t w = k == 0 ? q.x : (k == 1 ? q.y : (k == 2 ? q.z : q.w));
    return *reinterpret_cast<const __nv_bfloat162*>(&w);
  }
  __device__ __forceinline__ void set(int k, __nv_bfloat162 v) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(&v);
    if (k == 0) q.x = w;
    else if (k == 1) q.y = w;
    else if (k == 2) q.z = w;
    else q.w = w;
  }
  __device__ __forceinline__ void zero() { q = make_uint4(0u, 0u, 0u, 0u); }
};

__device__ __forceinline__ void unpack8(const V8& v, float (&f)[8]) {
  const uint32_t w[4] = {v.q.x, v.q.y, v.q.z, v.q.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {   // bf16 -> fp32 is a 16-bit shift
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ V8 pack8(const float (&f)[8]) {
  V8 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) v.set(i, __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]));
  return v;
}
__device__ __forceinline__ V8 ldg8(const void* p, long long vec_idx) {
  V8 v;
  v.q = __ldg(reinterpret_cast<const uint4*>(p) + vec_idx);
  return v;
}
__device__ __forceinline__ void stg8(void* p, long long vec_idx, const V8& v) {
  *(reinterpret_cast<uint4*>(p) + vec_idx) = v.q;
}

}  // namespace saicv
