// Fused multi-head attention on wgmma / TMA for sm_90a: forward and the two backward phases.
//
//   S = Q K^T * scale (+ key-padding mask);  P = softmax(S);  O = P V          (never materialised in HBM)
//
// One kernel family, templated on the score width DQK (q/k row length, multiple of 16, <= 256) and the
// value width DV (multiple of 16, <= 128); sequence lengths are runtime and tiled (64-row tiles, key / query
// blocks of 64), so the same code serves
//   ViT            hd 64, L = 197                     (classification/backbones/vit.py:62-80)
//   SAM encoder    hd 64/80, 14x14 windows (L = 196) and global attention (L = 4096); the decomposed
//                  rel-pos bias enters as extra score columns  [q | rel_h | rel_w] . [k | onehot_h | onehot_w]
//                  so DQK = hd + bias columns            (segment_anything/image_encoder.py:82-144,167-184)
//   DETR           hd 32, self attention with key-padding mask and cross attention Lq != Lk
//                                                        (detection/models/detr.py:54-56,103-109)
//
// CTA = 160 threads, persistent over (batch*head, row tile) work items:
//   warps 0..3  one consumer warpgroup: S = Q K^T by wgmma into registers (fragment layout, see ptx.cuh), softmax
//               in registers (a row is spread over the 4 lanes of a quad), bf16 P into 128B-swizzled shared memory
//               (the A operand of P V), O accumulated in registers
//   warp 4      TMA producer (one lane): the row tile once per item, column blocks through a 2-stage ring
#pragma once
#include "dropout_hash.cuh"
#include "ptx.cuh"

namespace saicv {

constexpr int kAttnThreads = 160;
constexpr int kAttnRows = 64;   // rows of a tile = the M of one wgmma
constexpr int kAttnCols = 64;   // keys (forward, backward phase A) / queries (phase B) per column block

struct AttnDrop {            // attention-probability dropout (thresh == 0: off), see dropout_hash.cuh
  uint32_t thresh, seed_lo, seed_hi;
  float scale;                // 1 / (1 - p)
  const unsigned long long* seed_base;   // device word added to the seed (nullable): fresh masks per CUDA-graph replay
};
// the effective seed words of this launch (one uniform global load when a device base is given)
__device__ __forceinline__ AttnDrop resolve_drop(const AttnDrop& d) {
  AttnDrop r = d;
  if (d.thresh != 0 && d.seed_base != nullptr) {
    const unsigned long long s = (((unsigned long long)d.seed_hi << 32) | d.seed_lo) + *d.seed_base;
    r.seed_lo = (uint32_t)s;
    r.seed_hi = (uint32_t)(s >> 32);
  }
  return r;
}

struct AttnParams {
  AttnDrop drop;
  int B, H, Lq, Lk;
  int num_q_tiles;          // ceil(Lq / 64)
  float scale_log2;         // softmax scale * log2(e)
  float scale;
  __nv_bfloat16* out;       // [b][row][h][DV] through strides (elements)
  long long o_sb, o_sh, o_sl;
  float* lse;               // [B][H][Lq]  log2 domain: m + log2(sum)
  const uint32_t* mask_bits;  // [B][mask_words] bit k%32 of word k/32 set = key k masked out; may be null
  int mask_words;
};

// S[64 x 64] = A[64 x D] * B[64 x D]^T, both operands K-major in 64-column chunks of 64 rows (8192 bytes apart)
template <int D>
__device__ __forceinline__ void wg_scores(float (&s)[32], uint32_t a_addr, uint32_t b_addr) {
#pragma unroll
  for (int k = 0; k < D / 16; ++k) {
    const uint32_t off = (k >> 2) * 8192 + (k & 3) * 32;
    wgmma_m64n64<0, 0>(s, make_smem_desc(a_addr + off, 16, 1024), make_smem_desc(b_addr + off, 16, 1024), k > 0 ? 1 : 0);
  }
}
// D[64 x N] += A[64 x 64] * B[64 x N]: A K-major (one 8192-byte tile written by the consumer threads), B MN-major
// (rows = reduction index, N contiguous) in 64-column chunks 8192 bytes apart
template <int N>
__device__ __forceinline__ void wg_accumulate(float (&d)[N / 2], uint32_t a_addr, uint32_t b_addr) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_m64<N, 0, 1>(d, make_smem_desc(a_addr + k * 32, 16, 1024), b_addr + k * 2048, 8192,
                       [](int n0) { return (uint32_t)((n0 >> 6) * 8192 + (n0 & 63) * 2); }, 1);
}

// Fragment coordinates of accumulator register i of an m64nN tile (ptx.cuh, wgmma): row (0..63) and column.
__device__ __forceinline__ int frag_row(int i, int warp, int lane) { return warp * 16 + (lane >> 2) + ((i & 2) ? 8 : 0); }
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }
// bf16 pair (row, col), (row, col + 1) into a 64-row x 64-column K-major tile, 128B-swizzled (col even)
__device__ __forceinline__ void store_pair(uint8_t* tile, int row, int col, float a, float b) {
  *reinterpret_cast<uint32_t*>(tile + row * 128 + ((((col >> 3) ^ (row & 7))) << 4) + (col & 7) * 2) = pack_bf16x2(a, b);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// 1024-byte aligned base of the dynamic shared memory (128B-swizzle atoms); every footprint reserves the slack
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~static_cast<uintptr_t>(1023));
}

template <int DQK, int DV>
struct AttnFwdCfg {
  static constexpr int NCQ = (DQK + 63) / 64, NCV = (DV + 63) / 64;
  static constexpr int QBYTES = NCQ * 8192, KBYTES = NCQ * 8192, VBYTES = NCV * 8192, PBYTES = 8192;
  static constexpr int kStages = 2;   // K / V ring depth
  static constexpr int kSmemBytes = 1024 + QBYTES + kStages * (KBYTES + VBYTES) + PBYTES + 256;
};

// Forward.  Online softmax per key block: m = running row maximum of the raw scores, O and l rescaled by
// 2^((m_old - m_new) * scale_log2) when it rises; P = exp2(s * scale_log2 - m * scale_log2).
template <int DQK, int DV, int MINB, bool DROP>
__global__ void __launch_bounds__(kAttnThreads, MINB)
attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  using Cfg = AttnFwdCfg<DQK, DV>;
  constexpr int BN = kAttnCols, NCQ = Cfg::NCQ, NCV = Cfg::NCV, kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::QBYTES;
  uint8_t* sV = sK + kStages * Cfg::KBYTES;
  uint8_t* sP = sV + kStages * Cfg::VBYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + Cfg::PBYTES);
  uint64_t* q_full = bars + 0;
  uint64_t* q_empty = bars + 1;
  uint64_t* k_full = bars + 2;              // [kStages]
  uint64_t* k_empty = k_full + kStages;
  uint64_t* v_full = k_empty + kStages;
  uint64_t* v_empty = v_full + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 4);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 4);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int nkb = (p.Lk + BN - 1) / BN;
  const int total = p.B * p.H * p.num_q_tiles;

  if (warp == 4) {
    // ================================================================ TMA producer
    if (lane == 0) {
      uint32_t it = 0, g = 0;  // work items done, key blocks issued (ring position)
      for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
        const int qt = w % p.num_q_tiles, bh = w / p.num_q_tiles, b = bh / p.H, h = bh % p.H;
        mbar_wait(q_empty, (it & 1) ^ 1);
        mbar_expect_tx(q_full, Cfg::QBYTES);
#pragma unroll
        for (int c = 0; c < NCQ; ++c) tma_load_4d(&tmQ, q_full, sQ + c * 8192, c * 64, qt * kAttnRows, h, b);
        for (int j = 0; j < nkb; ++j, ++g) {
          const int st = g % kStages;
          const uint32_t ph = (g / kStages) & 1;
          mbar_wait(&k_empty[st], ph ^ 1);
          mbar_expect_tx(&k_full[st], Cfg::KBYTES);
#pragma unroll
          for (int c = 0; c < NCQ; ++c) tma_load_4d(&tmK, &k_full[st], sK + st * Cfg::KBYTES + c * 8192, c * 64, j * BN, h, b);
          mbar_wait(&v_empty[st], ph ^ 1);
          mbar_expect_tx(&v_full[st], Cfg::VBYTES);
#pragma unroll
          for (int c = 0; c < NCV; ++c) tma_load_4d(&tmV, &v_full[st], sV + st * Cfg::VBYTES + c * 8192, c * 64, j * BN, h, b);
        }
      }
    }
    return;
  }
  // ================================================================ consumer warpgroup
  const AttnDrop drop = DROP ? resolve_drop(p.drop) : p.drop;
  uint32_t it = 0, g = 0;
  for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
    const int qt = w % p.num_q_tiles, bh = w / p.num_q_tiles, b = bh / p.H, h = bh % p.H;
    float o[DV / 2];
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows frag_row(0) and frag_row(2) of this thread
    mbar_wait(q_full, it & 1);
    for (int j = 0; j < nkb; ++j, ++g) {
      const int st = g % kStages;
      const uint32_t ph = (g / kStages) & 1;
      const int nvalid = min(BN, p.Lk - j * BN);
      float s[32];
      mbar_wait(&k_full[st], ph);
      wgmma_fence();
      wg_scores<DQK>(s, smem_u32(sQ), smem_u32(sK + st * Cfg::KBYTES));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&k_empty[st]);
        if (j == nkb - 1) mbar_arrive(q_empty);
      }
      // key padding / mask -> -inf, row maxima
      float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = frag_col(i, lane);
        bool dead = col >= nvalid;
        if (p.mask_bits) dead |= (__ldg(p.mask_bits + (long long)b * p.mask_words + ((j * BN + col) >> 5)) >> (col & 31)) & 1u;
        s[i] = dead ? -INFINITY : s[i];
        bm[(i >> 1) & 1] = fmaxf(bm[(i >> 1) & 1], s[i]);
      }
      float corr[2], msl[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float m_new = fmaxf(m[r], quad_max(bm[r]));
        corr[r] = m_new == -INFINITY ? 1.f : ex2_approx((m[r] - m_new) * p.scale_log2);
        msl[r] = m_new == -INFINITY ? 0.f : m_new * p.scale_log2;
        m[r] = m_new;
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        s[i] = ex2_approx(fmaf(s[i], p.scale_log2, -msl[(i >> 1) & 1]));
        rs[(i >> 1) & 1] += s[i];
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) l[r] = l[r] * corr[r] + quad_sum(rs[r]);
#pragma unroll
      for (int i = 0; i < DV / 2; ++i) o[i] *= corr[(i >> 1) & 1];
      if (DROP) {   // the row sum is that of the undropped probabilities; P V uses the dropped ones
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const uint32_t drow = (uint32_t)(bh * p.Lq + qt * kAttnRows + frag_row(i, warp, lane));
          s[i] = dropout_hash(drop.seed_lo, drop.seed_hi, drow, (uint32_t)(j * BN + frag_col(i, lane))) >= drop.thresh
                     ? s[i] * drop.scale : 0.f;
        }
      }
      named_bar_sync(1, 128);   // the previous block's P V has retired in every warp: the P tile may be overwritten
#pragma unroll
      for (int i = 0; i < 32; i += 2) store_pair(sP, frag_row(i, warp, lane), frag_col(i, lane), s[i], s[i + 1]);
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      mbar_wait(&v_full[st], ph);
      wgmma_fence_regs(o);
      wgmma_fence();
      wg_accumulate<DV>(o, smem_u32(sP), smem_u32(sV + st * Cfg::VBYTES));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[st]);
    }
    // ---- epilogue: normalise, store the rows and their log-sum-exp
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) inv[r] = l[r] > 0.f ? __fdividef(1.f, l[r]) : 0.f;
#pragma unroll
    for (int i = 0; i < DV / 2; i += 2) {
      const int qrow = qt * kAttnRows + frag_row(i, warp, lane);
      if (qrow < p.Lq) {
        __nv_bfloat16* orow = p.out + (long long)b * p.o_sb + (long long)h * p.o_sh + (long long)qrow * p.o_sl;
        *reinterpret_cast<uint32_t*>(orow + frag_col(i, lane)) = pack_bf16x2(o[i] * inv[(i >> 1) & 1], o[i + 1] * inv[(i >> 1) & 1]);
      }
    }
    if ((lane & 3) == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int qrow = qt * kAttnRows + frag_row(2 * r, warp, lane);
        if (qrow < p.Lq) p.lse[((long long)b * p.H + h) * p.Lq + qrow] = l[r] > 0.f ? m[r] * p.scale_log2 + log2f(l[r]) : -INFINITY;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
struct AttnBwdParams {
  AttnDrop drop;
  int B, H, Lq, Lk;
  int num_tiles;            // row tiles per (b, h): ceil(Lq / 64) in the dQ phase, ceil(Lk / 64) in the dK/dV phase
  float scale_log2, scale;
  const float* lse;         // [B][H][Lq]
  const float* delta;       // [B][H][Lq]  D = rowsum(dO * O)
  const uint32_t* mask_bits;
  int mask_words;
  __nv_bfloat16* d_out0;    // dQ (phase A) or dK (phase B)
  long long s0b, s0h, s0l;
  __nv_bfloat16* d_out1;    // dV (phase B)
  long long s1b, s1h, s1l;
  int dk_cols;              // phase B: leading columns of dK that are stored (<= DQK)
};

// Phase A (ROWS_ARE_KEYS = false): row tile = 64 queries, column blocks = 64 keys:
//     S = Q K^T, dP = dO V^T, dS = P (dP - D) scale, dQ += dS K              (dQ accumulates in registers)
// Phase B (ROWS_ARE_KEYS = true): row tile = 64 keys, column blocks = 64 queries:
//     S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q                  (dK, dV accumulate in registers)
// tmR0 / tmR1: the row-tile operands (A: Q, dO; B: K, V); tmC0 / tmC1: the column-block operands (A: K, V; B: Q, dO).
template <int DQK, int DV, bool ROWS_ARE_KEYS>
struct AttnBwdCfg {
  static constexpr int NCQ = (DQK + 63) / 64, NCV = (DV + 63) / 64;
  static constexpr int kStages = 2;
  static constexpr int R0BYTES = NCQ * 8192, R1BYTES = NCV * 8192;         // row tiles (64 rows)
  static constexpr int C0BYTES = NCQ * 8192, C1BYTES = NCV * 8192;         // column blocks (64 rows)
  static constexpr int ABYTES = 8192;                                        // one [64 x 64] bf16 A tile
  static constexpr int NA = ROWS_ARE_KEYS ? 2 : 1;
  static constexpr int kSmemBytes = 1024 + R0BYTES + R1BYTES + kStages * (C0BYTES + C1BYTES) + NA * ABYTES + 512 /*lse, delta*/ + 256;
};

template <int DQK, int DV, bool ROWS_ARE_KEYS, int MINB, bool DROP>
__global__ void __launch_bounds__(kAttnThreads, MINB)
attn_bwd_sm90_kernel(const __grid_constant__ CUtensorMap tmR0, const __grid_constant__ CUtensorMap tmR1,
                     const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ CUtensorMap tmC1,
                     const AttnBwdParams p) {
  using Cfg = AttnBwdCfg<DQK, DV, ROWS_ARE_KEYS>;
  constexpr int BN = kAttnCols, NCQ = Cfg::NCQ, NCV = Cfg::NCV, kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sR0 = smem;
  uint8_t* sR1 = sR0 + Cfg::R0BYTES;
  uint8_t* sC0 = sR1 + Cfg::R1BYTES;
  uint8_t* sC1 = sC0 + kStages * Cfg::C0BYTES;
  uint8_t* sA0 = sC1 + kStages * Cfg::C1BYTES;      // dS (phase A) / P^T (phase B)
  uint8_t* sA1 = sA0 + Cfg::ABYTES;                 // dS^T (phase B)
  float* sLse = reinterpret_cast<float*>(sA0 + Cfg::NA * Cfg::ABYTES);   // [2][64] phase B: lse / delta of the query block
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sLse) + 512);
  uint64_t* r_full = bars + 0;
  uint64_t* r_empty = bars + 1;
  uint64_t* c_full = bars + 2;            // [kStages]
  uint64_t* c_empty = c_full + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmR0);
    tma_prefetch_desc(&tmR1);
    tma_prefetch_desc(&tmC0);
    tma_prefetch_desc(&tmC1);
    mbar_init(r_full, 1);
    mbar_init(r_empty, 4);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&c_full[i], 1);
      mbar_init(&c_empty[i], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int Lrow = ROWS_ARE_KEYS ? p.Lk : p.Lq;     // length along the row tiles
  const int Lcol = ROWS_ARE_KEYS ? p.Lq : p.Lk;     // length along the column blocks
  const int ncb = (Lcol + BN - 1) / BN;
  const int total = p.B * p.H * p.num_tiles;

  if (warp == 4) {
    // ================================================================ TMA producer
    if (lane == 0) {
      uint32_t it = 0, g = 0;
      for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
        const int rt = w % p.num_tiles, bh = w / p.num_tiles, b = bh / p.H, h = bh % p.H;
        mbar_wait(r_empty, (it & 1) ^ 1);
        mbar_expect_tx(r_full, Cfg::R0BYTES + Cfg::R1BYTES);
#pragma unroll
        for (int c = 0; c < NCQ; ++c) tma_load_4d(&tmR0, r_full, sR0 + c * 8192, c * 64, rt * kAttnRows, h, b);
#pragma unroll
        for (int c = 0; c < NCV; ++c) tma_load_4d(&tmR1, r_full, sR1 + c * 8192, c * 64, rt * kAttnRows, h, b);
        for (int j = 0; j < ncb; ++j, ++g) {
          const int st = g % kStages;
          const uint32_t ph = (g / kStages) & 1;
          mbar_wait(&c_empty[st], ph ^ 1);
          mbar_expect_tx(&c_full[st], Cfg::C0BYTES + Cfg::C1BYTES);
#pragma unroll
          for (int c = 0; c < NCQ; ++c)
            tma_load_4d(&tmC0, &c_full[st], sC0 + st * Cfg::C0BYTES + c * 8192, c * 64, j * BN, h, b);
#pragma unroll
          for (int c = 0; c < NCV; ++c)
            tma_load_4d(&tmC1, &c_full[st], sC1 + st * Cfg::C1BYTES + c * 8192, c * 64, j * BN, h, b);
        }
      }
    }
    return;
  }
  // ================================================================ consumer warpgroup (registers: fragment layout)
  const AttnDrop drop = DROP ? resolve_drop(p.drop) : p.drop;
  const int tid = threadIdx.x;
  constexpr int NACC0 = ROWS_ARE_KEYS ? DV : DQK;   // dV (B) / dQ (A)
  constexpr int NACC1 = ROWS_ARE_KEYS ? DQK : 16;   // dK (B); unused in phase A
  uint32_t it = 0, g = 0;
  for (int w = blockIdx.x; w < total; w += gridDim.x, ++it) {
    const int rt = w % p.num_tiles, bh = w / p.num_tiles, b = bh / p.H, h = bh % p.H;
    int grow[2];
    bool row_dead[2];
    float lse_r[2] = {0.f, 0.f}, dl_r[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      grow[r] = rt * kAttnRows + frag_row(2 * r, warp, lane);   // query in phase A, key in phase B
      row_dead[r] = grow[r] >= Lrow;
      if (!ROWS_ARE_KEYS) {
        if (!row_dead[r]) {
          lse_r[r] = p.lse[(long long)bh * p.Lq + grow[r]];
          dl_r[r] = p.delta[(long long)bh * p.Lq + grow[r]];
        }
      } else if (p.mask_bits && !row_dead[r]) {
        row_dead[r] = (__ldg(p.mask_bits + (long long)b * p.mask_words + (grow[r] >> 5)) >> (grow[r] & 31)) & 1u;
      }
    }
    float acc0[NACC0 / 2], acc1[NACC1 / 2];
#pragma unroll
    for (int i = 0; i < NACC0 / 2; ++i) acc0[i] = 0.f;
#pragma unroll
    for (int i = 0; i < NACC1 / 2; ++i) acc1[i] = 0.f;
    mbar_wait(r_full, it & 1);
    for (int j = 0; j < ncb; ++j, ++g) {
      const int st = g % kStages;
      const uint32_t ph = (g / kStages) & 1;
      const int nvalid = min(BN, Lcol - j * BN);
      named_bar_sync(1, 128);   // the previous block's accumulate MMAs (A tiles) and lse / delta readers are done
      if (ROWS_ARE_KEYS) {
        // lse / delta of the 64 queries of this block -> shared memory
        const int q = j * BN + (tid & 63);
        sLse[tid] = q < p.Lq ? (tid < 64 ? p.lse : p.delta)[(long long)bh * p.Lq + q] : 0.f;
      }
      mbar_wait(&c_full[st], ph);
      const uint8_t* c0 = sC0 + st * Cfg::C0BYTES;
      const uint8_t* c1 = sC1 + st * Cfg::C1BYTES;
      float sv[32], dv[32];
      wgmma_fence();
      wg_scores<DQK>(sv, smem_u32(sR0), smem_u32(c0));
      wg_scores<DV>(dv, smem_u32(sR1), smem_u32(c1));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sv);
      wgmma_fence_regs(dv);
      if (ROWS_ARE_KEYS) named_bar_sync(1, 128);   // sLse written
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = (i >> 1) & 1;
        const int lc = frag_col(i, lane);
        float pp[2], ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = j * BN + lc + e;
          const float ls = ROWS_ARE_KEYS ? sLse[lc + e] : lse_r[r];
          const float dl = ROWS_ARE_KEYS ? sLse[64 + lc + e] : dl_r[r];
          pp[e] = ex2_approx(fmaf(sv[i + e], p.scale_log2, -ls));
          float dpv = dv[i + e];
          if (DROP) {
            // A~ = M A / (1 - p):  dS = A (M dP / (1 - p) - D);  dV uses A~ (phase B's P tile)
            const uint32_t qi = ROWS_ARE_KEYS ? (uint32_t)col : (uint32_t)grow[r];
            const uint32_t ki = ROWS_ARE_KEYS ? (uint32_t)grow[r] : (uint32_t)col;
            const bool keep = dropout_hash(drop.seed_lo, drop.seed_hi, (uint32_t)bh * (uint32_t)p.Lq + qi, ki) >= drop.thresh;
            dpv = keep ? dpv * drop.scale : 0.f;
            ds[e] = pp[e] * (dpv - dl);
            pp[e] = keep ? pp[e] * drop.scale : 0.f;
          } else {
            ds[e] = pp[e] * (dpv - dl);
          }
          bool dead = row_dead[r] || lc + e >= nvalid;
          if (!ROWS_ARE_KEYS && p.mask_bits)
            dead |= (__ldg(p.mask_bits + (long long)b * p.mask_words + (col >> 5)) >> (col & 31)) & 1u;
          pp[e] = dead ? 0.f : pp[e];
          ds[e] = dead ? 0.f : ds[e];
        }
        const int row = frag_row(i, warp, lane);
        if (ROWS_ARE_KEYS) {
          store_pair(sA0, row, lc, pp[0], pp[1]);
          store_pair(sA1, row, lc, ds[0], ds[1]);
        } else {
          store_pair(sA0, row, lc, ds[0], ds[1]);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      wgmma_fence();
      if (!ROWS_ARE_KEYS) {
        wg_accumulate<NACC0>(acc0, smem_u32(sA0), smem_u32(c0));   // dQ += dS K_j
      } else {
        wg_accumulate<NACC0>(acc0, smem_u32(sA0), smem_u32(c1));   // dV += P^T dO_i
        wg_accumulate<NACC1>(acc1, smem_u32(sA1), smem_u32(c0));   // dK += dS^T Q_i
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      __syncwarp();
      if (lane == 0) mbar_arrive(&c_empty[st]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(r_empty);
    // ---- store the accumulators (dQ, dK scaled by the softmax scale)
#pragma unroll
    for (int i = 0; i < NACC0 / 2; i += 2) {
      const int r = (i >> 1) & 1;
      if (grow[r] < Lrow) {
        const float sc = ROWS_ARE_KEYS ? 1.f : p.scale;
        __nv_bfloat16* dst = ROWS_ARE_KEYS
            ? p.d_out1 + (long long)b * p.s1b + (long long)h * p.s1h + (long long)grow[r] * p.s1l
            : p.d_out0 + (long long)b * p.s0b + (long long)h * p.s0h + (long long)grow[r] * p.s0l;
        *reinterpret_cast<uint32_t*>(dst + frag_col(i, lane)) = pack_bf16x2(acc0[i] * sc, acc0[i + 1] * sc);
      }
    }
    if (ROWS_ARE_KEYS) {
#pragma unroll
      for (int i = 0; i < NACC1 / 2; i += 2) {
        const int r = (i >> 1) & 1;
        const int col = frag_col(i, lane);
        if (grow[r] < Lrow && col < p.dk_cols) {
          __nv_bfloat16* dst = p.d_out0 + (long long)b * p.s0b + (long long)h * p.s0h + (long long)grow[r] * p.s0l;
          *reinterpret_cast<uint32_t*>(dst + col) = pack_bf16x2(acc1[i] * p.scale, acc1[i + 1] * p.scale);
        }
      }
    }
  }
}

}  // namespace saicv
