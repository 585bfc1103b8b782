// Counter-hash dropout shared by the elementwise dropout kernel (capi_detr.cu) and the attention kernels
// (attn_sm90.cuh): the keep decision of element (a, b) under a 64-bit seed is a pure function, so the backward
// pass recomputes the forward's mask instead of storing it.  keep <=> hash >= round(p * 2^32).
// tests/test_detr_gpu.py restates the same integer arithmetic in torch to inject identical masks into the oracle.
#pragma once
#include <cstdint>

namespace saicv {

__host__ __device__ __forceinline__ uint32_t dropout_hash(uint32_t seed_lo, uint32_t seed_hi, uint32_t a, uint32_t b) {
  uint32_t x = (a + seed_lo) * 0x9E3779B1u;
  x ^= (b + seed_hi) * 0x85EBCA77u;
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}

inline uint32_t dropout_threshold(float p) {
  const double t = (double)p * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}

}  // namespace saicv
