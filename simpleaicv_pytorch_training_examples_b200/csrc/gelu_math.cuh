// Exact-erf GELU terms shared by the GEMM epilogues (gemm_sm90.cuh) and the streaming kernels (capi_vit.cu).
//
//   Phi(x) = 0.5 (1 + erf(x / sqrt 2)),  phi(x) = exp(-x^2 / 2) / sqrt(2 pi);  gelu = x Phi,  gelu' = Phi + x phi
//
// erf by Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7, far below the bf16 resolution of the stored result):
//   1 - erf(z) = (a1 t + ... + a5 t^5) exp(-z^2),  t = 1 / (1 + p z),  z = |x| / sqrt 2
// The one exponential is shared with phi.  Both transcendental steps are single MUFU instructions on arguments that
// need no range handling: ex2.approx.ftz of a value <= 0 (underflow to 0 is the right answer) and rcp.approx.ftz of a
// value >= 1.  (__expf / __fdividef expand to 6 + 5 instructions with their range fix-ups; with them these terms cost
// ~30 instructions per element and made the fused epilogues - 8 warps per SM for 128 x 256 outputs per tile - the
// bottleneck of the ViT / SAM MLP data gradient.)  13 FMA-pipe + 2 MUFU instructions per element.
#pragma once
#include "ptx.cuh"

namespace saicv {

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void gelu_terms(float x, float& cdf, float& pdf) {
  const float e = ex2_approx((x * x) * -0.72134752044448170368f);            // exp(-x^2/2) = 2^(-x^2 log2(e) / 2)
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752440f, fabsf(x), 1.0f));
  const float poly = t * (0.254829592f + t * (-0.284496736f + t * (1.421413741f + t * (-1.453152027f + t * 1.061405429f))));
  const float h = 0.5f * (poly * e);                                           // (1 - erf(|x| / sqrt 2)) / 2 = Phi(-|x|)
  cdf = x >= 0.f ? 1.0f - h : h;
  pdf = 0.3989422804014327f * e;
}
__device__ __forceinline__ float gelu_erf(float x) {
  float cdf, pdf;
  gelu_terms(x, cdf, pdf);
  return x * cdf;
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float cdf, pdf;
  gelu_terms(x, cdf, pdf);
  return fmaf(x, pdf, cdf);
}

}  // namespace saicv
