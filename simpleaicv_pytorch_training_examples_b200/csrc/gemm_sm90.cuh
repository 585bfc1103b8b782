// Persistent, warp-specialised wgmma GEMM / implicit-GEMM convolution engine for sm_90a.
//
//   D[M, N] (+ split-K partials) = A[M, K] * B[N, K]^T     bf16 x bf16 -> fp32 (registers)
//
// One CTA per SM, 384 threads:
//   warp 0      TMA producer (one lane)        global -> 128B-swizzled smem ring
//   warps 1..3  idle (keep the consumers on aligned warpgroups)
//   warps 4..11 two consumer warpgroups; warpgroup h owns columns h*64 .. h*64+63 of the 128 x BN tile:
//               wgmma (two m64n64 row blocks) -> registers -> per-warp transpose through shared memory so that a
//               thread owns one row -> (bias/act/residual) -> smem -> TMA store
//
// Operand feeding modes (runtime, so that fprop / dgrad / wgrad of linear layers and of NHWC
// convolutions all go through this one kernel):
//   A_K2D    A is a row-major [M, K] matrix                      (linear fwd / dgrad, 1x1 conv)
//   A_IM2COL A is an NHWC activation tensor read with TMA im2col (conv fprop / dgrad)
//   A_MN2D   A is stored [K, M] (K = reduction over pixels)      (wgrad: dY^T)
//   A_IM2COL_MN A is an NHWC tensor read with TMA im2col, [pixels, C] (transposed conv wgrad dW^T = X^T dY, few filters;
//            VAR_PLAIN_F32 only)
//   B_K2D    B is a row-major [N, K] matrix                      (weights, fprop)
//   B_MN2D   B is stored [K, N]                                  (weights for dgrad, x for wgrad)
//   B_IM2COL B is an NHWC tensor read with TMA im2col, [pixels, C] (wgrad of a conv)
#pragma once
#include "gelu_math.cuh"
#include "ptx.cuh"

namespace saicv {

enum : int { A_K2D = 0, A_IM2COL = 1, A_MN2D = 2, A_IM2COL_MN = 3 };
enum : int { B_K2D = 0, B_MN2D = 2, B_IM2COL = 3 };
enum : int { EPI_BIAS = 1, EPI_RELU = 2, EPI_GELU = 4, EPI_DIRECT = 8, EPI_RESID = 16, EPI_RESID_BF16 = 32,
              EPI_MUL_DGELU = 64, EPI_ROW_SCALE = 128, EPI_STATS = 256, EPI_MUL_DRELU = 512, EPI_MASK_BITS = 1024 };

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 384;  // 4 control warps (TMA producer + 3 idle) + 8 consumer / epilogue warps
constexpr int kStoreBufBytes = 16384;  // one staging slice: 128 rows x 128 B
constexpr int kMaxStoreBufs = 3;       // staging slices per epilogue half (runtime 1..3, GemmParams::store_bufs)
constexpr int kSmemTotal = 232448;     // dynamic shared memory every launch asks for (227 KB)
constexpr int kXposeStride = 33;       // floats per row of a warp's transpose buffer (32 columns + 1: conflict-free rows)
constexpr int kXposeBytes = 8 * 32 * kXposeStride * 4;   // one 32 x 32 fp32 buffer per consumer warp
constexpr int kSmemBudget = kSmemTotal - 1024 /*align slack*/ - 512 /*barriers*/ - kXposeBytes;

// The split of shared memory between the operand ring and the epilogue staging slices is a launch
// parameter (capi_gemm.cu: pick_smem_split): long reductions want >= 4 ring stages and get one slice
// per half, short reductions (the epilogue-bound 1x1 convolutions, K = 64..256) trade ring stages
// for 2-3 slices so that a TMA store (and the TMA load of the next aux slice) is never waited for
// right after it was issued.
template <int BN>
struct GemmCfg {
  static constexpr int kStageBytes = BM * BK * 2 + BN * BK * 2;
  static constexpr int kStagesRaw = (kSmemBudget - 2 * kStoreBufBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;   // upper bound of the ring depth
  static constexpr int kSmemBytes = kSmemTotal;
  static_assert(BN == 64 || BN == 128, "a consumer warpgroup owns 64 columns: BN is 64 (one warpgroup) or 128 (two)");
  static constexpr int kConsumerWGs = BN / 64;
};

struct ConvGeom {
  // Geometry of the tensor that is read in im2col mode (A for fprop/dgrad, B for wgrad).
  int P, Q;          // output spatial extent (rows of the implicit GEMM = n*P*Q + p*Q + q)
  int stride;        // traversal stride
  int lc_h, lc_w;    // lower corner (= -pad for fprop/wgrad, pad-(R-1) for dgrad)
  int R, S;          // filter taps
  int cchunks;       // channels of the im2col tensor / 64
  int n_img;         // batch (used to push padding tiles out of bounds)
};

struct GemmParams {
  int M, N;            // output extent
  int num_kb;          // total 64-wide reduction blocks
  int kb_per_split;    // reduction blocks handled by one split
  int splits;
  int a_mode, b_mode;
  int flip_taps;       // dgrad: B tap index is mirrored
  int b_cin;           // dgrad/fprop: channels per tap in the weight matrix row (Cin)
  ConvGeom g;
  int epi_flags;
  int out_f32;         // 1: D is fp32, else bf16
  const float* bias;   // [N] or null
  const float* resid;  // fp32 [M, ldd] residual added in the epilogue (EPI_RESID) or null
  const void* resid_bf16;  // bf16 [M, ldd]: added (EPI_RESID_BF16); as pre-activation u, D *= gelu'(u) (EPI_MUL_DGELU); as ReLU output, D *= (r > 0) (EPI_MUL_DRELU)
  const float* row_scale;  // EPI_ROW_SCALE: D = resid + row_scale[row / rows_per_scale] * (acc + bias) (drop-path)
  int rows_per_scale;
  void* out;           // direct-store path
  long long ldd;       // leading dimension of D in elements
  long long split_stride;  // elements between split-K partial outputs
  int num_stages;      // smem ring depth actually used (<= GemmCfg::kStages)
  int store_bufs;      // staging slices per epilogue half (1..kMaxStoreBufs)
  int aux_tma;         // 1: the aux operand of the epilogue (resid when out_f32, resid_bf16 otherwise) has the
                       // output's element width and is brought in by TMA (tensor map tmR) INTO the staging
                       // slice, combined in place and stored from there; 0: per-thread global loads
  float* stats_partial;  // EPI_STATS: [gridDim.x][2][N] per-CTA column sums / sums of squares of the bf16 output
  const uint32_t* mask_bits;  // EPI_MASK_BITS: [M][N/32] ReLU mask (bit j of word w: column 32w + j); applied last as D *= bit
  int tile_rows;       // rows of D per work item (BM; the phase dgrad stores whole rows of the compact dy: (BM / Q) * Q)
  // Data gradient of a 3x3 / stride 2 / pad 1 convolution by output phase: dx pixel (2p+a, 2q+b) only receives dy at
  // (p, q) + {0, 1}^2 through a fixed subset of the taps, so each phase (a, b) is a stride-1 correlation over the compact
  // dy with 1, 2 or 4 taps (9 in all).  `phases` (1 otherwise) is the outermost work index; D is stored through a 5-D
  // map {c, b, q, a, n*P + p} over dx (capi_gemm.cu: saicv_conv_dgrad).
  int phases;
  int ph_out[4];       // (a << 1) | b of each phase, in work order
  int ph_taps[4];      // taps of each phase
  int ph_tab[4][4];    // per tap, in reduction order: weight tap (r*S + s) | dy row offset << 8 | dy column offset << 9
};

// Kernel variants: the epilogue's feature set is a compile-time mask, so that the common launches run a compact
// instruction stream (with every feature a run-time branch, branch resolution and instruction fetch take a large share of
// the issue slots of the short-reduction launches, whose pace the epilogue sets).  VAR_FULL and VAR_AUX spill a few
// hundred bytes at the 168-register cap of 384 threads (ptxas -v); the other variants do not spill.
//   VAR_FULL        every flag but EPI_MASK_BITS / output type at run time (GELU forward, EPI_DIRECT, per-thread aux loads)
//   VAR_PLAIN_BF16  bf16 output, optional bias / ReLU / BatchNorm statistics       (conv fprop, plain dgrad, Linear)
//   VAR_PLAIN_F32   fp32 output, optional bias                                       (split-K weight gradients, fp32 Linear)
//   VAR_AUX         aux operand by TMA (fp32 residual, bf16 addend / ReLU mask / GELU pre-activation), bias, row scale,
//                   1-bit ReLU mask (conv dgrad + shortcut gradient, masked by the previous residual block's output ReLU)
//   VAR_STATS_BF16  VAR_PLAIN_BF16 with the BatchNorm statistics taken by FOUR EXTRA WARPS (512 threads): the column sums of
//                   a staged slice cost ~2.8x the work of staging it (instruction count), so they are taken off the
//                   epilogue warps.  The stats warps read the slice from shared memory while the epilogue
//                   warps are already draining the next chunk (handshake: staged / stats-done mbarriers per slice).
//   VAR_PHASE_BF16  bf16 output, no epilogue operation: the stride-2 data gradient by output phase (GemmParams::phases), a
//                   variant of its own so that the other launches do not carry its work decomposition
enum : int { VAR_FULL = 0, VAR_PLAIN_BF16 = 1, VAR_PLAIN_F32 = 2, VAR_AUX = 3, VAR_STATS_BF16 = 4, VAR_PHASE_BF16 = 5 };
template <int VAR>
struct GemmVariant {
  static constexpr int kMask = VAR == VAR_FULL ? (0x7fffffff & ~EPI_MASK_BITS)
                               : (VAR == VAR_PLAIN_BF16 || VAR == VAR_STATS_BF16) ? (EPI_BIAS | EPI_RELU | EPI_STATS)
                               : VAR == VAR_PLAIN_F32 ? EPI_BIAS
                               : VAR == VAR_PHASE_BF16 ? 0
                               : (EPI_BIAS | EPI_ROW_SCALE | EPI_RESID | EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU |
                                  EPI_MASK_BITS);
  static constexpr int kOut = (VAR == VAR_PLAIN_BF16 || VAR == VAR_STATS_BF16 || VAR == VAR_PHASE_BF16) ? 1 : VAR == VAR_PLAIN_F32 ? 2 : 0;   // 0: run time, 1: bf16, 2: fp32
  static constexpr int kAux = VAR == VAR_FULL ? 0 : VAR == VAR_AUX ? 2 : 1;                // 0: run time, 1: never, 2: always by TMA
  static constexpr bool kStatsWarps = VAR == VAR_STATS_BF16;                               // statistics by warps 12..15
  static constexpr bool kPhases = VAR == VAR_PHASE_BF16;                                   // GemmParams::phases / tile_rows honoured
  static constexpr int kThreads = kStatsWarps ? kGemmThreads + 128 : kGemmThreads;
};

// Reduction of one tile by one consumer warpgroup: acc[blk] = rows blk*64 .. +63 x the warpgroup's 64 columns
// (`b_off`: byte offset of its first column in a B stage).  Both operand layouts put row / column 64 at +8192 bytes.
// A stage is handed back to the producer (one arrival per warp) once the wgmma group that read it has retired.
template <int BN, int TA, int TB>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[2][32], const uint8_t* sA, const uint8_t* sB, uint64_t* full_bar,
                                              uint64_t* empty_bar, int nstages, int& stage, uint32_t& phase, int kb0, int kb1,
                                              uint32_t b_off, int lane) {
  constexpr int kABytes = BM * BK * 2, kBBytes = BN * BK * 2;
  constexpr uint32_t a_lbo = TA ? 8192u : 16u, b_lbo = TB ? 8192u : 16u;
  constexpr uint32_t a_kstep = TA ? 2048u : 32u, b_kstep = TB ? 2048u : 32u;   // bytes per k16 step
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(sA + stage * kABytes);
    const uint32_t b_addr = smem_u32(sB + stage * kBBytes) + b_off;
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t db = make_smem_desc(b_addr + k * b_kstep, b_lbo, 1024);
      const int acc_in = (kb > kb0 || k > 0) ? 1 : 0;
      wgmma_m64n64<TA, TB>(acc[0], make_smem_desc(a_addr + k * a_kstep, a_lbo, 1024), db, acc_in);
      wgmma_m64n64<TA, TB>(acc[1], make_smem_desc(a_addr + 8192 + k * a_kstep, a_lbo, 1024), db, acc_in);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the group of the previous stage has retired: its operands may be overwritten
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = stage;
    if (++stage == nstages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc[0]);
  wgmma_fence_regs(acc[1]);
  if (prev >= 0) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
  }
}

// Operand A of the transposed conv weight gradient, im2col patches MN-major: the 64 output pixels kb*64 .. +63
// (reduction rows) x NCH 64-wide column chunks from chunk cb0 (chunk cb = tap * cchunks + channel chunk), chunk j at
// +8192 B, the same loads as B_IM2COL.  Chunks past the R*S taps read image n_img, out of bounds: zeros.
template <int NCH>
__device__ __forceinline__ void load_patch_chunks(const CUtensorMap* tm, uint64_t* bar, uint8_t* dst, const ConvGeom& g,
                                                  int cb0, int kb) {
  const int pix = kb * BK;
  const int PQ = g.P * g.Q;
  const int bn_ = pix / PQ;
  const int rem = pix - bn_ * PQ;
  const int pp = rem / g.Q;
  const int bh = pp * g.stride + g.lc_h;
  const int bw = (rem - pp * g.Q) * g.stride + g.lc_w;
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int cb = cb0 + j;
    const int tapj = cb / g.cchunks;
    const int ccj = cb - tapj * g.cchunks;
    const int rj = tapj / g.S;
    const int sj = tapj - rj * g.S;
    const bool valid = tapj < g.R * g.S;
    tma_load_im2col_4d(tm, bar, dst + j * 8192, ccj * 64, bw, bh, valid ? bn_ : g.n_img, (uint16_t)(valid ? sj : 0),
                       (uint16_t)(valid ? rj : 0));
  }
}

template <int BN, int VAR>
__global__ void __launch_bounds__(GemmVariant<VAR>::kThreads, 1)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                  const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kABytes = BM * BK * 2;
  constexpr int kBBytes = BN * BK * 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  using V = GemmVariant<VAR>;
  const int flags = p.epi_flags & V::kMask;          // bits outside the variant's mask are known zeros
  const bool out_f32 = V::kOut == 0 ? (p.out_f32 != 0) : (V::kOut == 2);
  const int nstages = p.num_stages;
  const bool do_stats = (flags & EPI_STATS) != 0;
  uint8_t* sA = smem;
  uint8_t* sB = smem + nstages * kABytes;
  uint8_t* sD = smem + nstages * Cfg::kStageBytes;
  const int NB = p.store_bufs;
  float* sStat = reinterpret_cast<float*>(sD + 2 * NB * kStoreBufBytes);  // [2][N] when EPI_STATS
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sD + 2 * NB * kStoreBufBytes + (do_stats ? ((8 * p.N + 15) & ~15) : 0));
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* aux_bar = empty_bar + kStages;   // [2 halves][kMaxStoreBufs]: aux slice landed in staging slice b
  uint64_t* staged_bar = aux_bar + 2 * kMaxStoreBufs;    // [2][kMaxStoreBufs] VAR_STATS_BF16: slice b of the half is staged
  uint64_t* sdone_bar = staged_bar + 2 * kMaxStoreBufs;  // [2][kMaxStoreBufs] the four stats warps have read slice b
  float* sXpose = reinterpret_cast<float*>(smem + kSmemTotal - 1024 - kXposeBytes);   // [8 warps][32][kXposeStride]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmD);
    if (V::kAux != 1 && p.aux_tma) tma_prefetch_desc(&tmR);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4 * Cfg::kConsumerWGs);   // one arrival per consumer warp
    }
    for (int i = 0; i < 2 * kMaxStoreBufs; ++i) {
      mbar_init(&aux_bar[i], 1);
      mbar_init(&staged_bar[i], 1);
      mbar_init(&sdone_bar[i], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int phases = V::kPhases ? p.phases : 1;
  const int tile_rows = V::kPhases ? p.tile_rows : BM;
  const int num_m = (p.M + tile_rows - 1) / tile_rows;
  const int num_n = (p.N + BN - 1) / BN;
  const int per_phase = num_m * num_n * p.splits;
  const int total = per_phase * phases;

  if (warp == 0) {
    // ================================================================ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int PQ = p.g.P * p.g.Q;
      for (int w = blockIdx.x; w < total; w += gridDim.x) {
        const int ph = V::kPhases ? w / per_phase : 0;
        const int wp = w - ph * per_phase;
        const int n_blk = wp % num_n;
        const int t = wp / num_n;
        const int m_blk = t % num_m;
        const int split = t / num_m;
        const int m0 = m_blk * tile_rows, n0 = n_blk * BN;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(phases > 1 ? p.ph_taps[ph] * p.g.cchunks : p.num_kb, kb0 + p.kb_per_split);
        // im2col base pixel of the A tile (fprop / dgrad): fixed for the whole tile
        int a_n = 0, a_h = 0, a_w = 0;
        if (p.a_mode == A_IM2COL) {
          a_n = m0 / PQ;
          const int rem = m0 - a_n * PQ;
          const int pp = rem / p.g.Q;
          a_h = pp * p.g.stride + p.g.lc_h;
          a_w = (rem - pp * p.g.Q) * p.g.stride + p.g.lc_w;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint64_t* bar = &full_bar[stage];
          mbar_expect_tx(bar, kABytes + kBBytes);
          uint8_t* a_dst = sA + stage * kABytes;
          uint8_t* b_dst = sB + stage * kBBytes;
          int tap = 0, cc = kb, r = 0, s = 0, tapb = 0;   // im2col offsets (r, s) of A, weight tap of B
          if (p.a_mode == A_IM2COL) {
            tap = kb / p.g.cchunks;
            cc = kb - tap * p.g.cchunks;
            if (phases > 1) {
              const int e = p.ph_tab[ph][tap];
              tapb = e & 0xff;
              r = (e >> 8) & 1;
              s = (e >> 9) & 1;
            } else {
              r = tap / p.g.S;
              s = tap - r * p.g.S;
              tapb = p.flip_taps ? (p.g.R * p.g.S - 1 - tap) : tap;
            }
          }
          // ---- A
          if (p.a_mode == A_K2D) {
            tma_load_2d(&tmA, bar, a_dst, kb * BK, m0);
          } else if (p.a_mode == A_IM2COL) {
            tma_load_im2col_4d(&tmA, bar, a_dst, cc * 64, a_w, a_h, a_n, (uint16_t)s, (uint16_t)r);
          } else if constexpr (VAR == VAR_PLAIN_F32) {
            if (p.a_mode == A_IM2COL_MN) {   // transposed conv wgrad: patches [pixels, R*S*C]
              load_patch_chunks<2>(&tmA, bar, a_dst, p.g, m0 / 64, kb);
            } else {  // A_MN2D
              tma_load_2d(&tmA, bar, a_dst, m0, kb * BK);
              tma_load_2d(&tmA, bar, a_dst + 8192, m0 + 64, kb * BK);
            }
          } else {  // A_MN2D: [K rows, M cols], two 64-wide column chunks
            tma_load_2d(&tmA, bar, a_dst, m0, kb * BK);
            tma_load_2d(&tmA, bar, a_dst + 8192, m0 + 64, kb * BK);
          }
          // ---- B
          if (p.b_mode == B_K2D) {
            tma_load_2d(&tmB, bar, b_dst, kb * BK, n0);
          } else if (p.b_mode == B_MN2D) {
            int col_base = 0, row = kb * BK;
            if (p.a_mode == A_IM2COL) {  // conv dgrad: weights [Cout, R*S*Cin]
              col_base = tapb * p.b_cin;
              row = cc * 64;
            }
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_2d(&tmB, bar, b_dst + j * 8192, col_base + n0 + j * 64, row);
          } else {  // B_IM2COL (wgrad): reduction rows = 64 output pixels starting at kb*64
            const int pix = kb * BK;
            const int bn_ = pix / PQ;
            const int rem = pix - bn_ * PQ;
            const int pp = rem / p.g.Q;
            const int bh = pp * p.g.stride + p.g.lc_h;
            const int bw = (rem - pp * p.g.Q) * p.g.stride + p.g.lc_w;
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) {
              const int cb = n0 / 64 + j;
              const int tapj = cb / p.g.cchunks;
              const int ccj = cb - tapj * p.g.cchunks;
              const int rj = tapj / p.g.S;
              const int sj = tapj - rj * p.g.S;
              const bool valid = tapj < p.g.R * p.g.S;
              tma_load_im2col_4d(&tmB, bar, b_dst + j * 8192, ccj * 64, bw, bh,
                                 valid ? bn_ : p.g.n_img, (uint16_t)(valid ? sj : 0),
                                 (uint16_t)(valid ? rj : 0));
            }
          }
          if (++stage == nstages) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4 && warp < 12) {
    // ================================================================ consumers: wgmma + epilogue
    // 8 warps: warpgroup `half` = e/4 reduces and drains columns half*64 .. +63 of every tile.  Warp e%4 of it holds
    // the accumulators of rows (e%4)*16 .. +15 and 64 + (e%4)*16 .. +15; after the reduction it transposes each
    // 32-column chunk through its own shared-memory buffer so that lane l owns one row.  Each half owns NB 16 KB staging slices
    // (128 rows x 128 B = 64 bf16 or 32 fp32 columns, 128B-swizzled) used round-robin and its own
    // TMA-store bulk groups: slice s is written while the store of slice s-1 is still reading.
    // With aux_tma the half's thread 0 also TMA-loads the aux operand of slice s+LA (LA = max(1, NB-1))
    // into the slice that store s-1 has released; every thread combines its own row in place.
    const int e = warp - 4;
    const int q = e & 3;
    const int half = e >> 2;
    const int gtid = threadIdx.x - 128 - half * 128;  // 0..127 inside the half
    const int row_in_tile = (lane < 16 ? 0 : 48) + q * 16 + lane;   // lanes 0..15: rows q*16.., 16..31: rows 64 + q*16..
    const int rsw = row_in_tile & 7;                  // 128B-swizzle phase of this thread's staging row
    const uint32_t bar_id = 1 + half;
    uint8_t* const sbase = sD + half * NB * kStoreBufBytes;
    uint64_t* const abar = aux_bar + half * kMaxStoreBufs;
    float* const xp = sXpose + e * 32 * kXposeStride;
    const bool direct = (flags & EPI_DIRECT) != 0;
    const bool aux_tma = V::kAux == 0 ? (p.aux_tma != 0) : (V::kAux == 2);
    // chunk (32 columns) range of this half: its 64 columns (one bf16 slice or two fp32 slices); none for half 1 of BN = 64
    constexpr int NCH = BN / 32;
    const int c_begin = half ? 2 : 0;
    const int c_end = half ? NCH : 2;
    const bool a_mn = VAR == VAR_PLAIN_F32 ? (p.a_mode == A_MN2D || p.a_mode == A_IM2COL_MN) : (p.a_mode == A_MN2D);
    const bool b_mn = (p.b_mode != B_K2D);
    int stage = 0;
    uint32_t phase = 0;
    const int spt = out_f32 ? (c_end - c_begin) : ((c_end - c_begin) >> 1);  // slices per tile of this half
    int bufi = 0;             // staging slice of the current output slice
    uint32_t aux_phase = 0;   // bit b: parity to wait for on abar[b]
    // aux prefetch cursor (thread 0 of the half): next slice to request = slice pf_j of work item pf_w
    long long pf_w = blockIdx.x;
    int pf_j = 0, pf_b = 0;
    auto request_aux = [&]() {
      if (pf_w < total) {
        const int n_blk2 = (int)(pf_w % num_n);
        const int m_blk2 = (int)((pf_w / num_n) % num_m);
        const int col = n_blk2 * BN + (out_f32 ? (c_begin + pf_j) * 32 : ((c_begin >> 1) + pf_j) * 64);
        mbar_expect_tx(&abar[pf_b], kStoreBufBytes);   // rows / columns past the matrix are zero-filled and counted
        tma_load_3d(&tmR, &abar[pf_b], sbase + pf_b * kStoreBufBytes, col, m_blk2 * tile_rows, 0);
      }
      if (++pf_j == spt) { pf_j = 0; pf_w += gridDim.x; }
      if (++pf_b == NB) pf_b = 0;
    };
    if (aux_tma && gtid == 0 && spt > 0) {
      const int la = NB > 1 ? NB - 1 : 1;
      for (int i = 0; i < la; ++i) request_aux();
    }
    constexpr int kStatBarThreads = V::kStatsWarps ? 384 : 256;
    uint32_t sd_phase = 0;     // VAR_STATS_BF16: bit b = parity of the stats-done barrier of staging slice b
    if (do_stats) {
      for (int j = threadIdx.x - 128; j < 2 * p.N; j += 256) sStat[j] = 0.f;
      named_bar_sync(3, kStatBarThreads);
    }
    for (int w = blockIdx.x; w < total; w += gridDim.x) {
      const int ph = V::kPhases ? w / per_phase : 0;
      const int wp = w - ph * per_phase;
      const int n_blk = wp % num_n;
      const int t = wp / num_n;
      const int m_blk = t % num_m;
      const int split = t / num_m;
      const int m0 = m_blk * tile_rows, n0 = n_blk * BN;
      const long long row = m0 + row_in_tile;
      if (c_begin >= c_end) continue;   // half 1 of a 64-wide tile: no columns
      float acc[2][32];
      {
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(phases > 1 ? p.ph_taps[ph] * p.g.cchunks : p.num_kb, kb0 + p.kb_per_split);
        const uint32_t b_off = half * 8192u;   // column 64 of a B stage (K-major: row 64; MN-major: second chunk)
        if (a_mn) gemm_mainloop<BN, 1, 1>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, kb0, kb1, b_off, lane);
        else if (b_mn) gemm_mainloop<BN, 0, 1>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, kb0, kb1, b_off, lane);
        else gemm_mainloop<BN, 0, 0>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, kb0, kb1, b_off, lane);
      }
#pragma unroll
      for (int ci = 0; ci < 2; ++ci) {
        const int c = c_begin + ci;
        const int col0 = n0 + c * 32;
        const int part = out_f32 ? 0 : ((c - c_begin) & 1);   // bf16: which 32-column half of the 64-column slice
        const bool s_begin = out_f32 || part == 0;
        const bool s_end = out_f32 || part == 1;
        uint8_t* const sbuf = sbase + bufi * kStoreBufBytes;
        uint8_t* const buf = sbuf + row_in_tile * 128;
        // operands of the epilogue are requested before the accumulator transpose so their latency overlaps it
        float bv = 0.f;
        if ((flags & EPI_BIAS) && col0 + lane < p.N) bv = __ldg(p.bias + col0 + lane);
        float4 rf[8];
        uint4 rb[4];
        const bool has_rf = (flags & EPI_RESID) && row < p.M;
        const bool has_rb = (flags & (EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU)) && row < p.M;
        float rscale = 1.f;
        if ((flags & EPI_ROW_SCALE) && row < p.M) rscale = __ldg(p.row_scale + row / p.rows_per_scale);
        uint32_t mbits = 0u;   // the mask word of this thread's row and 32 columns
        if ((flags & EPI_MASK_BITS) && row < p.M && col0 < p.N) mbits = __ldg(p.mask_bits + row * (p.N >> 5) + (col0 >> 5));
        if (!aux_tma) {
          if (has_rf) {
            const float4* rp = reinterpret_cast<const float4*>(p.resid + row * p.ldd + col0);
#pragma unroll
            for (int j = 0; j < 8; ++j) rf[j] = (col0 + 4 * j < p.N) ? __ldg(rp + j) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          if (has_rb) {
            const uint4* rp = reinterpret_cast<const uint4*>(
                reinterpret_cast<const __nv_bfloat16*>(p.resid_bf16) + row * p.ldd + col0);
#pragma unroll
            for (int j = 0; j < 4; ++j) rb[j] = (col0 + 8 * j < p.N) ? __ldg(rp + j) : make_uint4(0, 0, 0, 0);
          }
        }
        // columns c*32 .. +31 of the warp's 32 rows: fragment layout -> lane = row (see ptx.cuh, wgmma)
        __syncwarp();
#pragma unroll
        for (int blk = 0; blk < 2; ++blk) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = ci * 4 + jj;
            float* const dst = xp + (blk * 16 + (lane >> 2)) * kXposeStride + jj * 8 + 2 * (lane & 3);
            dst[0] = acc[blk][4 * j];
            dst[1] = acc[blk][4 * j + 1];
            dst[8 * kXposeStride] = acc[blk][4 * j + 2];
            dst[8 * kXposeStride + 1] = acc[blk][4 * j + 3];
          }
        }
        __syncwarp();
        float f[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] = xp[lane * kXposeStride + j];
        if (aux_tma) {
          // the aux slice was TMA-loaded into this staging slice; each thread reads its own (swizzled) row
          if (s_begin) mbar_wait(&abar[bufi], (aux_phase >> bufi) & 1u);
          if (out_f32) {
#pragma unroll
            for (int j = 0; j < 8; ++j) rf[j] = *reinterpret_cast<const float4*>(buf + ((j ^ rsw) << 4));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) rb[j] = *reinterpret_cast<const uint4*>(buf + (((part * 4 + j) ^ rsw) << 4));
          }
        }
        if (flags & EPI_BIAS) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] += __shfl_sync(0xffffffffu, bv, j);
        }
        if (flags & EPI_GELU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = gelu_erf(f[j]);
        }
        if (flags & EPI_RELU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.f);
        }
        if (flags & EPI_ROW_SCALE) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] *= rscale;
        }
        if (flags & EPI_RESID) {
          if (aux_tma || has_rf) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              f[4 * j] += rf[j].x; f[4 * j + 1] += rf[j].y; f[4 * j + 2] += rf[j].z; f[4 * j + 3] += rf[j].w;
            }
          }
        }
        if (flags & (EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU)) {
          if (aux_tma || has_rb) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t wv[4] = {rb[j].x, rb[j].y, rb[j].z, rb[j].w};
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const float2 ab = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wv[u]));
                if (flags & EPI_MUL_DGELU) {
                  f[8 * j + 2 * u] *= gelu_erf_grad(ab.x);
                  f[8 * j + 2 * u + 1] *= gelu_erf_grad(ab.y);
                } else if (flags & EPI_MUL_DRELU) {   // resid_bf16 = ReLU output: pass the gradient where it is > 0
                  f[8 * j + 2 * u] = ab.x > 0.f ? f[8 * j + 2 * u] : 0.f;
                  f[8 * j + 2 * u + 1] = ab.y > 0.f ? f[8 * j + 2 * u + 1] : 0.f;
                } else {
                  f[8 * j + 2 * u] += ab.x;
                  f[8 * j + 2 * u + 1] += ab.y;
                }
              }
            }
          }
        }
        if (flags & EPI_MASK_BITS) {
          // a multiply by 0 / 1, not a select: the zeros keep the sign a later (bf16(D) * relu'(out)) would give them
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] *= ((mbits >> j) & 1u) ? 1.f : 0.f;
        }
        if (direct) {
          if (row < p.M) {
            if (out_f32) {
              float* o = reinterpret_cast<float*>(p.out) + split * p.split_stride + row * p.ldd + col0;
#pragma unroll
              for (int j = 0; j < 32; j += 4)
                if (col0 + j < p.N)
                  *reinterpret_cast<float4*>(o + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
            } else {
              __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + split * p.split_stride +
                                 row * p.ldd + col0;
#pragma unroll
              for (int j = 0; j < 32; j += 8)
                if (col0 + j < p.N)
                  *reinterpret_cast<uint4*>(o + j) =
                      make_uint4(pack_bf16x2(f[j], f[j + 1]), pack_bf16x2(f[j + 2], f[j + 3]),
                                 pack_bf16x2(f[j + 4], f[j + 5]), pack_bf16x2(f[j + 6], f[j + 7]));
            }
          }
        } else {
          if (s_begin && !aux_tma) {
            // the store that last read this staging slice (NB slices ago) must have drained it (and the stats warps too)
            if (gtid == 0) {
              tma_store_wait_read_n(NB - 1);
              if (V::kStatsWarps && do_stats) {
                mbar_wait(&sdone_bar[half * kMaxStoreBufs + bufi], ((sd_phase >> bufi) & 1u) ^ 1u);
                sd_phase ^= (1u << bufi);
              }
            }
            named_bar_sync(bar_id, 128);
          }
          if (out_f32) {
            // one 128 B (32 x fp32) slice per TMA store
#pragma unroll
            for (int j = 0; j < 8; ++j)
              *reinterpret_cast<float4*>(buf + ((j ^ rsw) << 4)) =
                  make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
          } else {
            // bf16: two 32-column chunks make one 128 B (64 x bf16) slice
#pragma unroll
            for (int j = 0; j < 4; ++j)
              *reinterpret_cast<uint4*>(buf + (((part * 4 + j) ^ rsw) << 4)) =
                  make_uint4(pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                             pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
          }
          if (s_end) {
            fence_proxy_async_smem();
            named_bar_sync(bar_id, 128);
            const int scol = out_f32 ? col0 : col0 - 32;
            if (gtid == 0) {
              if (scol < p.N && phases > 1) {
                const int ab = p.ph_out[ph];
                asm volatile(
                    "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                        reinterpret_cast<uint64_t>(&tmD)),
                    "r"(smem_u32(sbuf)), "r"(scol), "r"(ab & 1), "r"(0), "r"(ab >> 1), "r"(m0 / p.g.Q)
                    : "memory");
              } else if (scol < p.N) {
                asm volatile(
                    "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                        reinterpret_cast<uint64_t>(&tmD)),
                    "r"(smem_u32(sbuf)), "r"(scol), "r"(m0), "r"(split)
                    : "memory");
              }
              tma_store_commit();
              if (aux_tma) {
                // the slice that store s-1 read becomes the landing buffer of aux slice s + LA
                tma_store_wait_read_n(NB > 1 ? 1 : 0);
                request_aux();
              }
            }
            if (V::kStatsWarps && do_stats) {
              if (gtid == 0) mbar_arrive(&staged_bar[half * kMaxStoreBufs + bufi]);   // hand the slice to the stats warps
            } else if (do_stats) {
              // BatchNorm statistics of the slice just staged (the bf16 values as stored), read back
              // from the swizzled buffer (conflict free: a warp reads the 128 contiguous bytes of one
              // row) concurrently with the TMA store of the same buffer.  Rows >= M / cols >= N are zero.
              // Fixed summation order (bit-reproducible, no atomics): warp wq of the half owns columns
              // wq*16..+15 of the slice for all 128 rows.  Lane l reads 8 bytes (4 columns) of row
              // i*8 + l/4: the 8 rows of one load hit 8 distinct swizzled 16-byte chunks, so the
              // 256-byte request is conflict free.  The 8 row-lanes are then folded by shuffles and
              // lanes 0..3 add to the accumulators they alone own.
              const int wq = gtid >> 5;
              const int piece = lane & 3;
              const int chunk = wq * 2 + (piece >> 1);
              const int r0 = lane >> 2;        // row of load i is i*8 + r0: its swizzle phase (row & 7) is r0 for every i
              const uint8_t* const sp = sbuf + r0 * 128 + ((chunk ^ r0) << 4) + (piece & 1) * 8;
              float sx[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const uint2 w2 = *reinterpret_cast<const uint2*>(sp + i * 1024);
                const float a0 = __uint_as_float(w2.x << 16), a1 = __uint_as_float(w2.x & 0xffff0000u);
                const float b0 = __uint_as_float(w2.y << 16), b1 = __uint_as_float(w2.y & 0xffff0000u);
                sx[0] += a0; sq[0] = fmaf(a0, a0, sq[0]);
                sx[1] += a1; sq[1] = fmaf(a1, a1, sq[1]);
                sx[2] += b0; sq[2] = fmaf(b0, b0, sq[2]);
                sx[3] += b1; sq[3] = fmaf(b1, b1, sq[3]);
              }
#pragma unroll
              for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  sx[j] += __shfl_xor_sync(0xffffffffu, sx[j], o);
                  sq[j] += __shfl_xor_sync(0xffffffffu, sq[j], o);
                }
              }
              const int gcol = scol + wq * 16 + piece * 4;
              if (lane < 4 && gcol < p.N) {  // N % 8 == 0: the 4 columns are valid together
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  sStat[gcol + j] += sx[j];
                  sStat[p.N + gcol + j] += sq[j];
                }
              }
            }
            aux_phase ^= (1u << bufi);
            if (++bufi == NB) bufi = 0;
          }
        }
      }
    }
    if (gtid == 0) tma_store_wait<0>();
    if (do_stats) {
      named_bar_sync(3, kStatBarThreads);
      float* dst = p.stats_partial + (long long)blockIdx.x * 2 * p.N;
      for (int j = threadIdx.x - 128; j < 2 * p.N; j += 256) dst[j] = sStat[j];
    }
  } else if (V::kStatsWarps && warp >= 12) {
    // ================================================================ statistics warps (VAR_STATS_BF16)
    // Warp wq owns columns wq*16 .. +15 of every staged 64-column slice of BOTH epilogue halves for all 128 rows (fixed
    // ownership and summation order: bit-reproducible, no atomics).  Lane l reads 8 bytes (4 columns) of row i*8 + l/4;
    // the 8 row-lanes are folded by shuffles and lanes 0..3 add to the shared-memory accumulators they alone own.
    if (do_stats) {
      const int wq = warp - 12;
      const int piece = lane & 3;
      const int chunk = wq * 2 + (piece >> 1);
      const int r0 = lane >> 2;
      const int soff = r0 * 128 + ((chunk ^ r0) << 4) + (piece & 1) * 8;
      constexpr int NCH = BN / 32;
      constexpr int split_at = 2 * ((BN / 64 + 1) / 2);
      constexpr int spt_h[2] = {split_at / 2, (NCH - split_at) / 2};
      int sb[2] = {0, 0};
      uint32_t st_phase[2] = {0u, 0u};
      named_bar_sync(3, 384);            // accumulators zeroed by the epilogue warps
      for (int w = blockIdx.x; w < total; w += gridDim.x) {
        const int n0 = (w % num_n) * BN;
#pragma unroll 1
        for (int j = 0; j < spt_h[0]; ++j) {
#pragma unroll 1
          for (int h = 0; h < 2; ++h) {
            if (j >= spt_h[h]) continue;
            const int b = sb[h];
            mbar_wait(&staged_bar[h * kMaxStoreBufs + b], (st_phase[h] >> b) & 1u);
            const uint8_t* const sp = sD + (h * NB + b) * kStoreBufBytes + soff;
            float sx[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const uint2 w2 = *reinterpret_cast<const uint2*>(sp + i * 1024);
              const float a0 = __uint_as_float(w2.x << 16), a1 = __uint_as_float(w2.x & 0xffff0000u);
              const float b0 = __uint_as_float(w2.y << 16), b1 = __uint_as_float(w2.y & 0xffff0000u);
              sx[0] += a0; sq[0] = fmaf(a0, a0, sq[0]);
              sx[1] += a1; sq[1] = fmaf(a1, a1, sq[1]);
              sx[2] += b0; sq[2] = fmaf(b0, b0, sq[2]);
              sx[3] += b1; sq[3] = fmaf(b1, b1, sq[3]);
            }
            // the slice is read: the epilogue may reuse it (after its TMA store has drained it too)
            __syncwarp();
            if (lane == 0) mbar_arrive(&sdone_bar[h * kMaxStoreBufs + b]);
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                sx[k] += __shfl_xor_sync(0xffffffffu, sx[k], o);
                sq[k] += __shfl_xor_sync(0xffffffffu, sq[k], o);
              }
            }
            const int gcol = n0 + ((h ? split_at : 0) / 2 + j) * 64 + wq * 16 + piece * 4;
            if (lane < 4 && gcol < p.N) {
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                sStat[gcol + k] += sx[k];
                sStat[p.N + gcol + k] += sq[k];
              }
            }
            st_phase[h] ^= (1u << b);
            sb[h] = (b + 1 == NB) ? 0 : b + 1;
          }
        }
      }
      named_bar_sync(3, 384);            // all slices accumulated: the epilogue warps write the partial row
    }
  }
}

}  // namespace saicv
