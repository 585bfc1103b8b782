// Multi-tensor optimizer step (SURVEY.md 8 f2): SGD-momentum and AdamW over ALL parameters of a model in ONE launch,
// with the refresh of the bf16 GEMM-operand copies (Linear [N][K], conv [K][R*S*Cp] tap-major) and the global-norm
// gradient clip fused in.  Replaces torch.optim.SGD / AdamW as the reference builds them (tools/utils.py:292-600; step at
// tools/scripts.py:209-248): torch's foreach path is 13 (SGD) / 45 (AdamW) launches per step followed, in this
// runtime, by one cast / re-layout kernel per weight.  HBM-bound: SGD 16 B/param (p, g, buf read; p, buf written) +
// 2 B/param shadow, AdamW 28 B/param + 2 B.
//
// Work decomposition: the host cuts every tensor into chunks of kChunk elements; block b processes chunk b
// (tensor id + offset from a device table), so big and tiny tensors share one grid.  Hyper-parameters live in DEVICE
// memory: a ring of SAICV_OPT_RING tables [slot][group][8] plus a device step counter that selects the slot
// (step % ring) and is advanced by a one-thread kernel after the update.  Launch arguments are therefore constants: the
// step is CUDA-graph safe with per-iteration learning rates - the host writes slot t % ring of a pinned copy before
// launching step t and a (captured) copy brings the ring in; the ring lets the host run up to ring-1 steps ahead.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/saicv_b200.h"
#include "host_util.h"

namespace saicv {
namespace {

constexpr int kOptThreads = 256;
constexpr int kChunk = SAICV_OPT_CHUNK;   // elements per block

// One parameter tensor (mirrors saicv_opt_tensor of the header, 72 bytes).
struct OptTensor {
  float* p;          // fp32 master parameter
  const float* g;    // fp32 gradient
  float* s1;         // SGD: momentum buffer; AdamW: exp_avg
  float* s2;         // AdamW: exp_avg_sq (unused for SGD)
  __nv_bfloat16* shadow;   // bf16 operand copy refreshed in the same pass, or null
  long long numel;
  int group;         // row of the hyper-parameter table
  int rs;            // shadow layout: 0 = same linear index; > 0 = conv weight [K][C][rs taps] -> [K][kpad], column tap*cp + c
  int c, cp, kpad;
  int step_idx;      // AdamW: index of the parameter's step count
};
static_assert(sizeof(OptTensor) == sizeof(saicv_opt_tensor) && sizeof(OptTensor) == 72, "saicv_opt_tensor layout");

__device__ __forceinline__ void write_shadow(const OptTensor& t, long long i, float v) {
  if (t.rs == 0) {
    t.shadow[i] = __float2bfloat16_rn(v);
  } else {
    const int crs = t.c * t.rs;
    const long long k = i / crs;
    const int rem = (int)(i - k * crs);
    const int c = rem / t.rs, tap = rem - c * t.rs;
    t.shadow[k * t.kpad + (long long)tap * t.cp + c] = __float2bfloat16_rn(v);
  }
}

// hyper[group] = {lr, weight_decay, momentum, nesterov, -, -, -, -}; clip[0] = gradient scale (1 when clipping is off)
template <bool kVec>
__device__ __forceinline__ void sgd_chunk(const OptTensor& t, long long base, int n, float lr, float wd, float mom, bool nesterov,
                                          float gs) {
  if (kVec) {
    float4* p4 = reinterpret_cast<float4*>(t.p + base);
    const float4* g4 = reinterpret_cast<const float4*>(t.g + base);
    float4* b4 = reinterpret_cast<float4*>(t.s1 + base);
    for (int i = threadIdx.x; i < n / 4; i += kOptThreads) {
      float4 p = p4[i], b = b4[i];
      const float4 g = g4[i];
      float pv[4] = {p.x, p.y, p.z, p.w}, bv[4] = {b.x, b.y, b.z, b.w};
      const float gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d = gv[j] * gs + wd * pv[j];
        bv[j] = mom * bv[j] + d;
        pv[j] -= lr * (nesterov ? d + mom * bv[j] : bv[j]);
      }
      p4[i] = make_float4(pv[0], pv[1], pv[2], pv[3]);
      b4[i] = make_float4(bv[0], bv[1], bv[2], bv[3]);
      if (t.shadow) {
#pragma unroll
        for (int j = 0; j < 4; ++j) write_shadow(t, base + 4 * i + j, pv[j]);
      }
    }
  } else {
    for (int i = threadIdx.x; i < n; i += kOptThreads) {
      float p = t.p[base + i];
      const float d = t.g[base + i] * gs + wd * p;
      const float b = mom * t.s1[base + i] + d;
      p -= lr * (nesterov ? d + mom * b : b);
      t.p[base + i] = p;
      t.s1[base + i] = b;
      if (t.shadow) write_shadow(t, base + i, p);
    }
  }
}

__global__ void __launch_bounds__(kOptThreads)
multi_sgd_kernel(const OptTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index,
                 const float* __restrict__ hyper, int n_groups, const int* __restrict__ step, const float* __restrict__ clip) {
  const OptTensor t = tensors[chunk_tensor[blockIdx.x]];
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  const float* h = hyper + ((long long)(*step % SAICV_OPT_RING) * n_groups + t.group) * 8;
  const float lr = h[0], wd = h[1], mom = h[2];
  const bool nesterov = h[3] != 0.f;
  const float gs = clip ? clip[0] : 1.f;
  const bool vec = ((reinterpret_cast<uintptr_t>(t.p + base) | reinterpret_cast<uintptr_t>(t.g + base) |
                     reinterpret_cast<uintptr_t>(t.s1 + base)) & 15) == 0 && (n & 3) == 0;
  if (vec) sgd_chunk<true>(t, base, n, lr, wd, mom, nesterov, gs);
  else sgd_chunk<false>(t, base, n, lr, wd, mom, nesterov, gs);
}

// AdamW exactly as torch.optim.AdamW (decoupled decay first): hyper[group] = {lr, weight_decay, beta1, beta2, eps, -, -, -}.
// The bias corrections come from the parameter's own step count t = steps[step_idx] + 1, which advances only in the steps
// that have its gradient (torch skips a parameter whose .grad is None), and are computed in double as torch does on the host.
__device__ __forceinline__ void adamw_elem(float& p, float g, float& m, float& v, float lr, float wd, float b1, float b2, float eps,
                                           float step_size, float bc2s) {
  p *= 1.f - lr * wd;
  m = m + (g - m) * (1.f - b1);                 // torch: exp_avg.lerp_(grad, 1 - beta1)
  v = b2 * v + (1.f - b2) * g * g;
  const float denom = sqrtf(v) / bc2s + eps;
  p -= step_size * (m / denom);
}

__global__ void __launch_bounds__(kOptThreads)
multi_adamw_kernel(const OptTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index,
                   const float* __restrict__ hyper, int n_groups, const int* __restrict__ step, const float* __restrict__ clip,
                   const int* __restrict__ steps) {
  const OptTensor t = tensors[chunk_tensor[blockIdx.x]];
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  const float* h = hyper + ((long long)(*step % SAICV_OPT_RING) * n_groups + t.group) * 8;
  const float lr = h[0], wd = h[1], b1 = h[2], b2 = h[3], eps = h[4];
  const int st = steps[t.step_idx] + 1;
  const float step_size = (float)((double)lr / (1.0 - pow((double)b1, st)));   // torch: lr / (1 - beta1^t)
  const float bc2s = (float)sqrt(1.0 - pow((double)b2, st));                   // torch: (1 - beta2^t) ** 0.5
  const float gs = clip ? clip[0] : 1.f;
  const bool vec = ((reinterpret_cast<uintptr_t>(t.p + base) | reinterpret_cast<uintptr_t>(t.g + base) |
                     reinterpret_cast<uintptr_t>(t.s1 + base) | reinterpret_cast<uintptr_t>(t.s2 + base)) & 15) == 0 && (n & 3) == 0;
  if (vec) {
    float4* p4 = reinterpret_cast<float4*>(t.p + base);
    const float4* g4 = reinterpret_cast<const float4*>(t.g + base);
    float4* m4 = reinterpret_cast<float4*>(t.s1 + base);
    float4* v4 = reinterpret_cast<float4*>(t.s2 + base);
    for (int i = threadIdx.x; i < n / 4; i += kOptThreads) {
      float4 p = p4[i], m = m4[i], v = v4[i];
      const float4 g = g4[i];
      adamw_elem(p.x, g.x * gs, m.x, v.x, lr, wd, b1, b2, eps, step_size, bc2s);
      adamw_elem(p.y, g.y * gs, m.y, v.y, lr, wd, b1, b2, eps, step_size, bc2s);
      adamw_elem(p.z, g.z * gs, m.z, v.z, lr, wd, b1, b2, eps, step_size, bc2s);
      adamw_elem(p.w, g.w * gs, m.w, v.w, lr, wd, b1, b2, eps, step_size, bc2s);
      p4[i] = p; m4[i] = m; v4[i] = v;
      if (t.shadow) {
        const float pv[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) write_shadow(t, base + 4 * i + j, pv[j]);
      }
    }
  } else {
    for (int i = threadIdx.x; i < n; i += kOptThreads) {
      float p = t.p[base + i], m = t.s1[base + i], v = t.s2[base + i];
      adamw_elem(p, t.g[base + i] * gs, m, v, lr, wd, b1, b2, eps, step_size, bc2s);
      t.p[base + i] = p; t.s1[base + i] = m; t.s2[base + i] = v;
      if (t.shadow) write_shadow(t, base + i, p);
    }
  }
}

// Advances the step count of every parameter of the table (those with a gradient) and the ring step.
__global__ void adamw_advance_kernel(const OptTensor* __restrict__ tensors, int n_tensors, int* __restrict__ steps,
                                     int* __restrict__ step) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_tensors) steps[tensors[i].step_idx] += 1;
  if (i == 0) *step += 1;
}

// Global gradient norm, deterministic: per-chunk sums of squares, then one block folds them in chunk order and writes
// clip = {min(1, max_norm / (norm + 1e-6)), norm}   (torch.nn.utils.clip_grad_norm_'s coefficient, NaN when the norm is).
__global__ void __launch_bounds__(kOptThreads)
multi_sqnorm_kernel(const OptTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index,
                    float* __restrict__ partial) {
  const OptTensor t = tensors[chunk_tensor[blockIdx.x]];
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kOptThreads) {
    const float g = t.g[base + i];
    s += g * g;
  }
  __shared__ float red[kOptThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < kOptThreads / 32; ++i) tot += red[i];
    partial[blockIdx.x] = tot;
  }
}

__global__ void __launch_bounds__(kOptThreads)
clip_coef_kernel(const float* __restrict__ partial, int n, float max_norm, float* __restrict__ clip) {
  __shared__ double red[kOptThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kOptThreads) s += (double)partial[i];   // fixed assignment of chunks to threads
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = kOptThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(red[0]);
    const float c = max_norm / (norm + 1e-6f);
    clip[0] = isnan(c) ? c : fminf(1.f, c);   // a NaN norm scales every gradient to NaN, as torch.clamp keeps it
    clip[1] = norm;
  }
}

__global__ void opt_advance_kernel(int* step) { *step += 1; }

// ---- Muon (tools/muon_optimizer.py of the reference; optim.FusedMuon).  A row of saicv_muon_tensor goes with each
// OptTensor row: s1 is the momentum buffer (Muon rows) or moment1 (AdamW rows), s2 moment2.  Muon rows own a bf16 slot
// [min(r, c)][ld] of the Newton-Schulz buffer holding X (transposed when r > c, as the reference does).
struct MuonTensor {
  long long slot;   // element offset of the slot; < 0: AdamW row
  int rows, cols;   // 2-D view of the parameter: [shape[0], numel / shape[0]]
  int ld;           // columns of the slot
  int transposed;   // slot = X^T (rows > cols)
  int chunk0, nchunks;   // chunks of this tensor in launch order (norm partials)
  int step_idx;     // AdamW rows: per-parameter step counter
  float adj;        // 0.2 * sqrt(max(shape[0], shape[1]))
};
static_assert(sizeof(MuonTensor) == sizeof(saicv_muon_tensor) && sizeof(MuonTensor) == 40, "saicv_muon_tensor layout");

__device__ __forceinline__ long long muon_slot_index(const MuonTensor& m, long long i) {
  const long long r = i / m.cols, c = i - r * m.cols;
  return m.slot + (m.transposed ? c * m.ld + r : r * m.ld + c);
}

__device__ __forceinline__ float block_sum(float s, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < kOptThreads / 32; ++i) tot += red[i];
  return tot;
}

// hyper[group] = {lr, weight_decay, momentum, nesterov, beta1, beta2, eps, -}
// buf = momentum * buf + g; u = nesterov ? g + momentum * buf : buf; partial[chunk] = sum of bf16(u)^2 over the chunk.
__global__ void __launch_bounds__(kOptThreads)
muon_momentum_kernel(const OptTensor* __restrict__ tensors, const MuonTensor* __restrict__ muon,
                     const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index, const float* __restrict__ hyper,
                     int n_groups, const int* __restrict__ step, const float* __restrict__ clip, float* __restrict__ partial) {
  const int ti = chunk_tensor[blockIdx.x];
  if (muon[ti].slot < 0) return;
  const OptTensor t = tensors[ti];
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  const float* h = hyper + ((long long)(*step % SAICV_OPT_RING) * n_groups + t.group) * 8;
  const float mom = h[2];
  const bool nesterov = h[3] != 0.f;
  const float gs = clip ? clip[0] : 1.f;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kOptThreads) {
    const float g = t.g[base + i] * gs;
    const float b = mom * t.s1[base + i] + g;
    t.s1[base + i] = b;
    const float u = __bfloat162float(__float2bfloat16_rn(nesterov ? g + mom * b : b));
    s = fmaf(u, u, s);
  }
  __shared__ float red[kOptThreads / 32];
  const float tot = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

// X = bf16(u / (||bf16(u)||_F + 1e-7)) into the slot; the norm folds the tensor's chunk partials in a fixed order, so every
// block of a tensor computes the same value.
__global__ void __launch_bounds__(kOptThreads)
muon_cast_kernel(const OptTensor* __restrict__ tensors, const MuonTensor* __restrict__ muon,
                 const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index, const float* __restrict__ hyper,
                 int n_groups, const int* __restrict__ step, const float* __restrict__ clip, const float* __restrict__ partial,
                 __nv_bfloat16* __restrict__ ns) {
  const int ti = chunk_tensor[blockIdx.x];
  const MuonTensor m = muon[ti];
  if (m.slot < 0) return;
  const OptTensor t = tensors[ti];
  __shared__ double dred[kOptThreads];
  double ds = 0.0;
  for (int i = threadIdx.x; i < m.nchunks; i += kOptThreads) ds += (double)partial[m.chunk0 + i];
  dred[threadIdx.x] = ds;
  __syncthreads();
  for (int o = kOptThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) dred[threadIdx.x] += dred[threadIdx.x + o];
    __syncthreads();
  }
  const float inv = 1.f / ((float)sqrt(dred[0]) + 1e-7f);
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  const float* h = hyper + ((long long)(*step % SAICV_OPT_RING) * n_groups + t.group) * 8;
  const float mom = h[2];
  const bool nesterov = h[3] != 0.f;
  const float gs = clip ? clip[0] : 1.f;
  for (int i = threadIdx.x; i < n; i += kOptThreads) {
    const float b = t.s1[base + i];
    const float u = __bfloat162float(__float2bfloat16_rn(nesterov ? t.g[base + i] * gs + mom * b : b));
    ns[muon_slot_index(m, base + i)] = __float2bfloat16_rn(u * inv);
  }
}

// Muon rows: p = p (1 - lr wd) - lr adj U.  AdamW rows (the reference's formula, not torch's AdamW): moments by lerp,
// p = p (1 - lr wd) - (lr sqrt(bc2) / bc1) m / (eps + sqrt(v)) with the parameter's own step count t = steps[idx] + 1.
__global__ void __launch_bounds__(kOptThreads)
muon_apply_kernel(const OptTensor* __restrict__ tensors, const MuonTensor* __restrict__ muon,
                  const int* __restrict__ chunk_tensor, const int* __restrict__ chunk_index, const float* __restrict__ hyper,
                  int n_groups, const int* __restrict__ step, const float* __restrict__ clip,
                  const __nv_bfloat16* __restrict__ ns, const int* __restrict__ adam_steps) {
  const int ti = chunk_tensor[blockIdx.x];
  const OptTensor t = tensors[ti];
  const MuonTensor m = muon[ti];
  const long long base = (long long)chunk_index[blockIdx.x] * kChunk;
  const int n = (int)min((long long)kChunk, t.numel - base);
  const float* h = hyper + ((long long)(*step % SAICV_OPT_RING) * n_groups + t.group) * 8;
  const float lr = h[0], wd = h[1], b1 = h[4], b2 = h[5], eps = h[6];
  const float decay = 1.f - lr * wd;
  if (m.slot >= 0) {
    const float a = lr * m.adj;
    for (int i = threadIdx.x; i < n; i += kOptThreads) {
      const float p = t.p[base + i] * decay - a * __bfloat162float(ns[muon_slot_index(m, base + i)]);
      t.p[base + i] = p;
      if (t.shadow) write_shadow(t, base + i, p);
    }
    return;
  }
  const int st = adam_steps[m.step_idx] + 1;
  const double bc1 = 1.0 - pow((double)b1, st), bc2 = 1.0 - pow((double)b2, st);
  const float a = (float)((double)lr * sqrt(bc2) / bc1);
  const float gs = clip ? clip[0] : 1.f;
  for (int i = threadIdx.x; i < n; i += kOptThreads) {
    const float g = t.g[base + i] * gs;
    float mv = t.s1[base + i], vv = t.s2[base + i];
    mv = mv + (g - mv) * (1.f - b1);
    vv = vv + (g * g - vv) * (1.f - b2);
    const float p = t.p[base + i] * decay - a * (mv / (eps + sqrtf(vv)));
    t.p[base + i] = p;
    t.s1[base + i] = mv;
    t.s2[base + i] = vv;
    if (t.shadow) write_shadow(t, base + i, p);
  }
}

// Advances the step count of every AdamW row of the table (parameters with a gradient) and the ring step.
__global__ void muon_advance_kernel(const MuonTensor* __restrict__ muon, int n_tensors, int* __restrict__ adam_steps,
                                    int* __restrict__ step) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_tensors && muon[i].slot < 0) adam_steps[muon[i].step_idx] += 1;
  if (i == 0) *step += 1;
}

}  // namespace
}  // namespace saicv

using namespace saicv;
#define ST reinterpret_cast<cudaStream_t>(stream)

extern "C" {

int saicv_opt_chunk(void) { return kChunk; }

int saicv_multi_tensor_sgd(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                           const float* hyper, int n_groups, int* step, const float* clip, void* stream) {
  if (n_chunks <= 0) return 0;
  multi_sgd_kernel<<<n_chunks, kOptThreads, 0, ST>>>(reinterpret_cast<const OptTensor*>(tensors), chunk_tensor, chunk_index, hyper,
                                                     n_groups, step, clip);
  if (check_launch("multi_sgd_kernel")) return 1;
  opt_advance_kernel<<<1, 1, 0, ST>>>(step);
  return check_launch("opt_advance_kernel");
}

int saicv_multi_tensor_adamw(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks, int n_tensors,
                             const float* hyper, int n_groups, int* step, const float* clip, int* steps, void* stream) {
  if (n_chunks <= 0) return 0;
  const OptTensor* t = reinterpret_cast<const OptTensor*>(tensors);
  multi_adamw_kernel<<<n_chunks, kOptThreads, 0, ST>>>(t, chunk_tensor, chunk_index, hyper, n_groups, step, clip, steps);
  if (check_launch("multi_adamw_kernel")) return 1;
  adamw_advance_kernel<<<(n_tensors + 255) / 256, 256, 0, ST>>>(t, n_tensors, steps, step);
  return check_launch("adamw_advance_kernel");
}

int saicv_multi_tensor_clip_coef(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                                 float max_norm, float* partial, float* clip, void* stream) {
  if (n_chunks <= 0) return set_error("saicv_multi_tensor_clip_coef: no tensors");
  multi_sqnorm_kernel<<<n_chunks, kOptThreads, 0, ST>>>(reinterpret_cast<const OptTensor*>(tensors), chunk_tensor, chunk_index, partial);
  if (check_launch("multi_sqnorm_kernel")) return 1;
  clip_coef_kernel<<<1, kOptThreads, 0, ST>>>(partial, n_chunks, max_norm, clip);
  return check_launch("clip_coef_kernel");
}

int saicv_muon_prep(const void* tensors, const void* muon, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                    const float* hyper, int n_groups, const int* step, const float* clip, float* partial, void* ns,
                    void* stream) {
  if (n_chunks <= 0) return 0;
  const OptTensor* t = reinterpret_cast<const OptTensor*>(tensors);
  const MuonTensor* m = reinterpret_cast<const MuonTensor*>(muon);
  muon_momentum_kernel<<<n_chunks, kOptThreads, 0, ST>>>(t, m, chunk_tensor, chunk_index, hyper, n_groups, step, clip, partial);
  if (check_launch("muon_momentum_kernel")) return 1;
  muon_cast_kernel<<<n_chunks, kOptThreads, 0, ST>>>(t, m, chunk_tensor, chunk_index, hyper, n_groups, step, clip, partial,
                                                     reinterpret_cast<__nv_bfloat16*>(ns));
  return check_launch("muon_cast_kernel");
}

int saicv_muon_apply(const void* tensors, const void* muon, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                     int n_tensors, const float* hyper, int n_groups, int* step, const float* clip, const void* ns,
                     int* adam_steps, void* stream) {
  if (n_chunks <= 0) return 0;
  const MuonTensor* m = reinterpret_cast<const MuonTensor*>(muon);
  muon_apply_kernel<<<n_chunks, kOptThreads, 0, ST>>>(reinterpret_cast<const OptTensor*>(tensors), m, chunk_tensor, chunk_index,
                                                      hyper, n_groups, step, clip,
                                                      reinterpret_cast<const __nv_bfloat16*>(ns), adam_steps);
  if (check_launch("muon_apply_kernel")) return 1;
  muon_advance_kernel<<<(n_tensors + 255) / 256, 256, 0, ST>>>(m, n_tensors, adam_steps, step);
  return check_launch("muon_advance_kernel");
}

}  // extern "C"
