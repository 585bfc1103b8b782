// Persistent, warp-specialised wgmma GEMM / implicit-GEMM convolution engine for sm_90a.
//
//   D[M, N] (+ split-K partials) = A[M, K] * B[N, K]^T     bf16 x bf16 -> fp32 (registers)
//
// One CTA per SM, 384 threads:
//   warp 0      TMA producer (one lane)        global -> 128B-swizzled smem ring
//   warps 1..3  idle (keep the consumers on aligned warpgroups)
//   warps 4..11 two consumer warpgroups; warpgroup h owns rows h*64 .. h*64+63 and all BN columns of the 128 x BN tile:
//               wgmma (one m64nBN per k16 step) -> registers -> (bias/act/residual) in the accumulator fragment
//               layout -> stmatrix / 8-byte stores into an smem slice shared by both warpgroups -> TMA store by one thread
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
enum : int { EPI_BIAS = 1, EPI_RELU = 2, EPI_RESID = 16, EPI_RESID_BF16 = 32,
              EPI_MUL_DGELU = 64, EPI_ROW_SCALE = 128, EPI_STATS = 256, EPI_MUL_DRELU = 512, EPI_MASK_BITS = 1024,
              EPI_AXPBY = 2048 };

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 384;  // 4 control warps (TMA producer + 3 idle) + 8 consumer / epilogue warps
constexpr int kStoreBufBytes = 16384;  // one staging slice: 128 rows x 128 B
constexpr int kMaxStoreBufs = 3;       // GemmParams::store_bufs (runtime 1..3): the tile's staging pool is 2 * store_bufs slices
constexpr int kSmemTotal = 232448;     // dynamic shared memory every launch asks for (227 KB)
constexpr int kSmemBudget = kSmemTotal - 1024 /*align slack*/ - 512 /*barriers*/;

// The split of shared memory between the operand ring and the epilogue staging slices is a launch
// parameter (capi_gemm.cu: pick_smem_split): long reductions want >= 4 ring stages and get two
// slices, short reductions (the epilogue-bound 1x1 convolutions, K = 64..256) trade ring stages
// for 4-6 slices so that a TMA store (and the TMA load of the next aux slice) is never waited for
// right after it was issued.
template <int BN>
struct GemmCfg {
  static constexpr int kStageBytes = BM * BK * 2 + BN * BK * 2;
  static constexpr int kStagesRaw = (kSmemBudget - 2 * kStoreBufBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;   // upper bound of the ring depth
  static constexpr int kSmemBytes = kSmemTotal;
  static_assert(BN == 64 || BN == 128, "a consumer warpgroup reduces 64 rows x BN columns with one m64nBN wgmma: BN is 64 or 128");
  static constexpr int kConsumerWGs = 2;   // rows 0..63 and 64..127 of every tile
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
  long long ldd;       // leading dimension of D (and of the aux operand) in elements
  int num_stages;      // smem ring depth actually used (<= GemmCfg::kStages)
  int store_bufs;      // 1..kMaxStoreBufs: the epilogue rotates through 2 * store_bufs staging slices
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
  // VAR_NS: `batch` same-shape matrices stacked in one buffer; the matrix is the outermost work index and the third
  // coordinate of the 3-D operand, aux and output maps.  EPI_AXPBY: D = alpha * acc + beta * aux.
  int batch;
  float alpha, beta;
};

// Kernel variants: the epilogue's feature set is a compile-time mask, so that the common launches run a compact
// instruction stream (with every feature a run-time branch, branch resolution and instruction fetch take a large share of
// the issue slots of the short-reduction launches, whose pace the epilogue sets).  No variant spills (ptxas -v); VAR_FULL
// at BN = 128 sits at the 168-register cap of 384 threads.
//   VAR_FULL        every flag but EPI_MASK_BITS / EPI_STATS / output type at run time (per-thread aux loads)
//   VAR_PLAIN_BF16  bf16 output, optional bias / ReLU                                (conv fprop, plain dgrad, Linear)
//   VAR_PLAIN_F32   fp32 output, optional bias                                       (split-K weight gradients, fp32 Linear)
//   VAR_AUX         aux operand by TMA (fp32 residual, bf16 addend / ReLU mask / GELU pre-activation), bias, row scale,
//                   1-bit ReLU mask (conv dgrad + shortcut gradient, masked by the previous residual block's output ReLU)
//   VAR_STATS_BF16  VAR_PLAIN_BF16 with the BatchNorm statistics taken by FOUR EXTRA WARPS (512 threads): the column sums of
//                   a staged slice cost ~2.8x the work of staging it (instruction count), so they are taken off the
//                   epilogue warps.  The stats warps read the slice from shared memory while the epilogue
//                   warps are already draining the next chunk (handshake: staged / stats-done mbarriers per slice).
//   VAR_PHASE_BF16  bf16 output, no epilogue operation: the stride-2 data gradient by output phase (GemmParams::phases), a
//                   variant of its own so that the other launches do not carry its work decomposition
//   VAR_NS          bf16 output over a batch of matrices (GemmParams::batch), optional D = alpha * acc + beta * aux with a
//                   bf16 aux operand by TMA: the Newton-Schulz products of the Muon optimizer (capi_gemm.cu: saicv_ns_gemm)
enum : int { VAR_FULL = 0, VAR_PLAIN_BF16 = 1, VAR_PLAIN_F32 = 2, VAR_AUX = 3, VAR_STATS_BF16 = 4, VAR_PHASE_BF16 = 5, VAR_NS = 6 };
template <int VAR>
struct GemmVariant {
  static constexpr int kMask = VAR == VAR_FULL ? (0x7fffffff & ~(EPI_MASK_BITS | EPI_STATS))
                               : VAR == VAR_PLAIN_BF16 ? (EPI_BIAS | EPI_RELU)
                               : VAR == VAR_STATS_BF16 ? (EPI_BIAS | EPI_RELU | EPI_STATS)
                               : VAR == VAR_PLAIN_F32 ? EPI_BIAS
                               : VAR == VAR_PHASE_BF16 ? 0
                               : VAR == VAR_NS ? EPI_AXPBY
                               : (EPI_BIAS | EPI_ROW_SCALE | EPI_RESID | EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU |
                                  EPI_MASK_BITS);
  static constexpr int kOut = (VAR == VAR_PLAIN_BF16 || VAR == VAR_STATS_BF16 || VAR == VAR_PHASE_BF16 || VAR == VAR_NS) ? 1 : VAR == VAR_PLAIN_F32 ? 2 : 0;   // 0: run time, 1: bf16, 2: fp32
  static constexpr int kAux = (VAR == VAR_FULL || VAR == VAR_NS) ? 0 : VAR == VAR_AUX ? 2 : 1;   // 0: run time, 1: never, 2: always by TMA
  static constexpr bool kStatsWarps = VAR == VAR_STATS_BF16;                               // statistics by warps 12..15
  static constexpr bool kPhases = VAR == VAR_PHASE_BF16;                                   // GemmParams::phases / tile_rows honoured
  static constexpr bool kBatch = VAR == VAR_NS;                                            // GemmParams::batch honoured
  static constexpr int kThreads = kStatsWarps ? kGemmThreads + 128 : kGemmThreads;
};

// Reduction of one tile by one consumer warpgroup: acc = its 64 rows (`a_off`: byte offset of the first one in an A
// stage; both operand layouts put row 64 at +8192 bytes) x all BN columns, one m64nBN wgmma per k16 step.  A K-major B
// stage is BN rows of 128 B; an MN-major one is BN / 64 chunks of 64 columns 8192 B apart, which is the descriptor's LBO.
// A stage is handed back to the producer (one arrival per warp) once the wgmma group that read it has retired.
template <int BN, int TA, int TB>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[BN / 2], const uint8_t* sA, const uint8_t* sB, uint64_t* full_bar,
                                              uint64_t* empty_bar, int nstages, int& stage, uint32_t& phase, int kb0, int kb1,
                                              uint32_t a_off, int lane) {
  constexpr int kABytes = BM * BK * 2, kBBytes = BN * BK * 2;
  constexpr uint32_t a_lbo = TA ? 8192u : 16u, b_lbo = TB ? 8192u : 16u;
  constexpr uint32_t a_kstep = TA ? 2048u : 32u, b_kstep = TB ? 2048u : 32u;   // bytes per k16 step
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(sA + stage * kABytes) + a_off;
    const uint32_t b_addr = smem_u32(sB + stage * kBBytes);
    wgmma_fence_regs(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t da = make_smem_desc(a_addr + k * a_kstep, a_lbo, 1024);
      const uint64_t db = make_smem_desc(b_addr + k * b_kstep, b_lbo, 1024);
      const int acc_in = (kb > kb0 || k > 0) ? 1 : 0;
      if constexpr (BN == 128) wgmma_m64n128<TA, TB>(acc, da, db, acc_in);
      else wgmma_m64n64<TA, TB>(acc, da, db, acc_in);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the group of the previous stage has retired: its operands may be overwritten
    wgmma_fence_regs(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = stage;
    if (++stage == nstages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (prev >= 0) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
  }
}

// Patch loads of a conv weight gradient (B_IM2COL, and A of the transposed product, A_IM2COL_MN): k-block kb is the 64
// output pixels kb*64 .. +63 (reduction rows) x up to two 64-wide column chunks from chunk cb0 (chunk cb = tap * cchunks
// + channel chunk), chunk j at +8192 B.  Chunks past the R*S taps read image n_img, out of bounds: zeros.  The column
// chunks are decoded once per work item and the pixel is stepped by 64 per k-block, so that the single producer lane
// issues no integer division per k-block (it requests every stage of the ring).
struct PatchWalk {
  int n, pp, pq;        // output pixel kb*64: image, row, column
  int dp, dq;           // 64 pixels = dp rows + dq columns
  int cc[2], r[2], s[2];
  bool valid[2];
  __device__ __forceinline__ void init(const ConvGeom& g, int cb0, int kb0) {
    const int pix = kb0 * BK, PQ = g.P * g.Q;
    n = pix / PQ;
    const int rem = pix - n * PQ;
    pp = rem / g.Q;
    pq = rem - pp * g.Q;
    dp = BK / g.Q;
    dq = BK - dp * g.Q;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int cb = cb0 + j;
      const int tap = cb / g.cchunks;
      cc[j] = cb - tap * g.cchunks;
      valid[j] = tap < g.R * g.S;
      r[j] = valid[j] ? tap / g.S : 0;
      s[j] = valid[j] ? tap - r[j] * g.S : 0;
    }
  }
  template <int NCH>
  __device__ __forceinline__ void load(const CUtensorMap* tm, uint64_t* bar, uint8_t* dst, const ConvGeom& g) const {
    const int bh = pp * g.stride + g.lc_h;
    const int bw = pq * g.stride + g.lc_w;
#pragma unroll
    for (int j = 0; j < NCH; ++j)
      tma_load_im2col_4d(tm, bar, dst + j * 8192, cc[j] * 64, bw, bh, valid[j] ? n : g.n_img, (uint16_t)s[j],
                         (uint16_t)r[j]);
  }
  __device__ __forceinline__ void step(const ConvGeom& g) {
    pq += dq;
    pp += dp;
    if (pq >= g.Q) { pq -= g.Q; ++pp; }
    while (pp >= g.P) { pp -= g.P; ++n; }
  }
};


// One work item: the output phase (VAR_PHASE_BF16) or matrix of the batch (VAR_NS), else 0; the first row and column of
// its tile; its split of the reduction and the k-blocks [kb0, kb1) of that split.
struct GemmTile {
  int ph, m0, n0, split, kb0, kb1;
};

// The work decomposition of a launch, the one place every warp role decodes a work item from.  Item w runs the n-block
// fastest, then the m-block, then the split, with the phase (or the matrix of the batch) outermost; CTA b takes items
// b, b + gridDim.x, ...  The producer and the consumers must agree on [kb0, kb1): both step the ring's mbarrier parities
// once per k-block.  The host counts the same items for the grid (capi_gemm.cu: gemm_grid), which is also the number of
// partial rows VAR_STATS_BF16 writes.
template <int BN, int VAR>
struct GemmSchedule {
  const GemmParams& p;
  int phases, tile_rows;   // GemmParams::phases / tile_rows where the variant honours them, else 1 / BM
  int num_m, num_n, per_phase, total;

  __device__ __forceinline__ explicit GemmSchedule(const GemmParams& params)
      : p(params),
        phases(GemmVariant<VAR>::kPhases ? params.phases : 1),
        tile_rows(GemmVariant<VAR>::kPhases ? params.tile_rows : BM),
        num_m((params.M + tile_rows - 1) / tile_rows),
        num_n((params.N + BN - 1) / BN),
        per_phase(num_m * num_n * params.splits),
        total(per_phase * phases * (GemmVariant<VAR>::kBatch ? params.batch : 1)) {}

  __device__ __forceinline__ GemmTile tile(int w) const {
    GemmTile t;
    t.ph = (GemmVariant<VAR>::kPhases || GemmVariant<VAR>::kBatch) ? w / per_phase : 0;
    const int wp = w - t.ph * per_phase;
    const int n_blk = wp % num_n;
    const int mt = wp / num_n;
    const int m_blk = mt % num_m;
    t.split = mt / num_m;
    t.m0 = m_blk * tile_rows;
    t.n0 = n_blk * BN;
    t.kb0 = t.split * p.kb_per_split;
    t.kb1 = min(phases > 1 ? p.ph_taps[t.ph] * p.g.cchunks : p.num_kb, t.kb0 + p.kb_per_split);
    return t;
  }
};

// TMA producer (one lane of warp 0): requests every k-block of the CTA's work items into the operand ring.
template <int BN, int VAR>
__device__ __forceinline__ void gemm_producer(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p,
                                              const GemmSchedule<BN, VAR>& sched, uint8_t* sA, uint8_t* sB,
                                              uint64_t* full_bar, uint64_t* empty_bar) {
  constexpr int kABytes = BM * BK * 2;
  constexpr int kBBytes = BN * BK * 2;
  const int nstages = p.num_stages;
  int stage = 0;
  uint32_t phase = 0;
  const int PQ = p.g.P * p.g.Q;
  for (int w = blockIdx.x; w < sched.total; w += gridDim.x) {
    const GemmTile t = sched.tile(w);
    // im2col base pixel of the A tile (fprop / dgrad): fixed for the whole tile
    int a_n = 0, a_h = 0, a_w = 0;
    if (p.a_mode == A_IM2COL) {
      a_n = t.m0 / PQ;
      const int rem = t.m0 - a_n * PQ;
      const int pp = rem / p.g.Q;
      a_h = pp * p.g.stride + p.g.lc_h;
      a_w = (rem - pp * p.g.Q) * p.g.stride + p.g.lc_w;
    }
    // (tap, channel chunk) of k-block kb = tap * cchunks + cc, and the tap's filter offsets (r, s): divided out once
    // per work item and stepped per k-block, so that the single producer lane issues no integer division per
    // k-block (it requests every stage of the ring, so its instruction count per k-block paces short-K convolutions)
    int tap = 0, cc = 0, r = 0, s = 0;
    if (p.a_mode == A_IM2COL) {
      tap = t.kb0 / p.g.cchunks;
      cc = t.kb0 - tap * p.g.cchunks;
      r = tap / p.g.S;
      s = tap - r * p.g.S;
    }
    const bool patches = p.b_mode == B_IM2COL || (VAR == VAR_PLAIN_F32 && p.a_mode == A_IM2COL_MN);
    PatchWalk pw;
    if (patches) pw.init(p.g, p.b_mode == B_IM2COL ? t.n0 / 64 : t.m0 / 64, t.kb0);
    for (int kb = t.kb0; kb < t.kb1; ++kb) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      uint64_t* bar = &full_bar[stage];
      mbar_expect_tx(bar, kABytes + kBBytes);
      uint8_t* a_dst = sA + stage * kABytes;
      uint8_t* b_dst = sB + stage * kBBytes;
      int ar = r, as = s, tapb = 0;   // im2col offsets (ar, as) of A, weight tap of B
      if (p.a_mode == A_IM2COL) {
        if (sched.phases > 1) {
          const int e = p.ph_tab[t.ph][tap];
          tapb = e & 0xff;
          ar = (e >> 8) & 1;
          as = (e >> 9) & 1;
        } else {
          tapb = p.flip_taps ? (p.g.R * p.g.S - 1 - tap) : tap;
        }
      }
      if constexpr (GemmVariant<VAR>::kBatch) {   // A K-major; B K-major or MN-major; coordinate 2 = matrix
        tma_load_3d(tmA, bar, a_dst, kb * BK, t.m0, t.ph);
        if (p.b_mode == B_K2D) {
          tma_load_3d(tmB, bar, b_dst, kb * BK, t.n0, t.ph);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_3d(tmB, bar, b_dst + j * 8192, t.n0 + j * 64, kb * BK, t.ph);
        }
        if (++stage == nstages) { stage = 0; phase ^= 1; }
        continue;
      }
      // ---- A
      if (p.a_mode == A_K2D) {
        tma_load_2d(tmA, bar, a_dst, kb * BK, t.m0);
      } else if (p.a_mode == A_IM2COL) {
        tma_load_im2col_4d(tmA, bar, a_dst, cc * 64, a_w, a_h, a_n, (uint16_t)as, (uint16_t)ar);
      } else if (VAR == VAR_PLAIN_F32 && p.a_mode == A_IM2COL_MN) {   // transposed conv wgrad: patches [pixels, R*S*C]
        pw.load<2>(tmA, bar, a_dst, p.g);
      } else {  // A_MN2D: [K rows, M cols], two 64-wide column chunks
        tma_load_2d(tmA, bar, a_dst, t.m0, kb * BK);
        tma_load_2d(tmA, bar, a_dst + 8192, t.m0 + 64, kb * BK);
      }
      // ---- B
      if (p.b_mode == B_K2D) {
        tma_load_2d(tmB, bar, b_dst, kb * BK, t.n0);
      } else if (p.b_mode == B_MN2D) {
        int col_base = 0, row = kb * BK;
        if (p.a_mode == A_IM2COL) {  // conv dgrad: weights [Cout, R*S*Cin]
          col_base = tapb * p.b_cin;
          row = cc * 64;
        }
#pragma unroll
        for (int j = 0; j < BN / 64; ++j)
          tma_load_2d(tmB, bar, b_dst + j * 8192, col_base + t.n0 + j * 64, row);
      } else {  // B_IM2COL (wgrad): reduction rows = 64 output pixels starting at kb*64
        pw.load<BN / 64>(tmB, bar, b_dst, p.g);
      }
      if (++stage == nstages) { stage = 0; phase ^= 1; }
      if (patches) pw.step(p.g);
      if (p.a_mode == A_IM2COL && ++cc == p.g.cchunks) {
        cc = 0;
        ++tap;
        if (++s == p.g.S) { s = 0; ++r; }
      }
    }
  }
}

// Consumer warpgroups (warps 4..11, `e` = warp - 4): wgmma mainloop and epilogue of every work item of the CTA.
// 8 warps: warpgroup `half` = e/4 reduces and drains rows half*64 .. +63 of every tile, all BN columns.  Warp e%4 of it
// holds the accumulators of rows half*64 + (e%4)*16 .. +15 in the wgmma fragment layout (ptx.cuh): lane l has rows
// l/4 and l/4 + 8 of them, column pairs 8j + 2*(l%4) + {0, 1}.  The epilogue runs in that layout and writes straight
// into the staging slices: bf16 by stmatrix (one 16 x 16 block per x4), fp32 by 8-byte stores; a bf16 aux operand
// comes back in the same layout by ldmatrix.  The tile's 2*NB 16 KB staging slices (128 rows x 128 B = 64 bf16 or 32
// fp32 columns, 128B-swizzled) are used round-robin in ascending column order; both warpgroups write their rows of the
// same slice, one 256-thread barrier closes it and the first consumer thread issues its TMA store: slice s is written
// while the stores of earlier slices still read.  With aux_tma that thread also TMA-loads the aux operand of slice
// s+LA (LA = 2*NB - 1) into the slice that store s-1 has released; every thread combines its own fragments in place.
template <int BN, int VAR>
__device__ __forceinline__ void gemm_consumer(const CUtensorMap* tmD, const CUtensorMap* tmR, const GemmParams& p,
                                              const GemmSchedule<BN, VAR>& sched, const uint8_t* sA, const uint8_t* sB,
                                              uint8_t* sD, float* sStat, uint64_t* full_bar, uint64_t* empty_bar,
                                              uint64_t* aux_bar, uint64_t* staged_bar, uint64_t* sdone_bar, int e,
                                              int lane) {
  using V = GemmVariant<VAR>;
  const int flags = p.epi_flags & V::kMask;          // bits outside the variant's mask are known zeros
  const bool out_f32 = V::kOut == 0 ? (p.out_f32 != 0) : (V::kOut == 2);
  const int q = e & 3;
  const int half = e >> 2;
  const bool leader = threadIdx.x == 128;           // issues the TMA stores and the aux requests of the tile
  const int r_lo = half * 64 + q * 16 + (lane >> 2);   // this thread's rows of the tile: r_lo and r_lo + 8
  const int cp = 2 * (lane & 3);                    // first column of this thread's pair in each 8-column group
  // stmatrix / ldmatrix: lane l addresses row (l/8 & 1)*8 + l%8 of the warp's 16, 16-byte unit (l/16) of a 16-column
  // block; fp32: the 8-byte half (l & 1) of unit (l/2 & 1) of an 8-column group, rows r_lo and r_lo + 8.  Both rows of a
  // lane share the 128B-swizzle phase (r & 7) with the row it addresses.
  const uint32_t mrow = (uint32_t)(half * 64 + q * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * 128u;
  const int mu = lane >> 4;
  const int sw = lane & 7;
  const int fsw = lane >> 2;
  const uint32_t frow = (uint32_t)r_lo * 128u + (uint32_t)(lane & 1) * 8u;
  const int fu = (lane >> 1) & 1;
  const uint32_t bar_id = 1;
  const int NBT = 2 * p.store_bufs;                 // staging slices of the tile
  const bool aux_tma = V::kAux == 0 ? (p.aux_tma != 0) : (V::kAux == 2);
  constexpr int NCH = BN / 32;                      // 32-column chunks of a tile
  const bool a_mn = VAR == VAR_PLAIN_F32 ? (p.a_mode == A_MN2D || p.a_mode == A_IM2COL_MN) : (p.a_mode == A_MN2D);
  const bool b_mn = (p.b_mode != B_K2D);
  const int nstages = p.num_stages;
  int stage = 0;
  uint32_t phase = 0;
  const int spt = out_f32 ? NCH : (NCH >> 1);       // slices per tile
  int bufi = 0;             // staging slice of the current output slice
  uint32_t aux_phase = 0;   // bit b: parity to wait for on aux_bar[b]
  // aux prefetch cursor (leader): next slice to request = slice pf_j of work item pf_w
  int pf_w = blockIdx.x;
  int pf_j = 0, pf_b = 0;
  auto request_aux = [&]() {
    if (pf_w < sched.total) {
      const GemmTile t = sched.tile(pf_w);
      const int col = t.n0 + pf_j * (out_f32 ? 32 : 64);
      mbar_expect_tx(&aux_bar[pf_b], kStoreBufBytes);   // rows / columns past the matrix are zero-filled and counted
      tma_load_3d(tmR, &aux_bar[pf_b], sD + pf_b * kStoreBufBytes, col, t.m0, V::kBatch ? t.ph : 0);
    }
    if (++pf_j == spt) { pf_j = 0; pf_w += gridDim.x; }
    if (++pf_b == NBT) pf_b = 0;
  };
  if (aux_tma && leader) {
    for (int i = 0; i < NBT - 1; ++i) request_aux();
  }
  uint32_t sd_phase = 0;     // VAR_STATS_BF16: bit b = parity of the stats-done barrier of staging slice b
  if (V::kStatsWarps) {
    for (int j = threadIdx.x - 128; j < 2 * p.N; j += 256) sStat[j] = 0.f;
    named_bar_sync(3, 384);   // with the four stats warps
  }
  for (int w = blockIdx.x; w < sched.total; w += gridDim.x) {
    const GemmTile t = sched.tile(w);
    const long long row0 = t.m0 + r_lo;               // rows of fragment halves h = 0, 1: row0 + 8h
    const bool in0 = row0 < p.M, in1 = row0 + 8 < p.M;
    float acc[BN / 2];
    {
      const uint32_t a_off = half * 8192u;   // row 64 of an A stage (K-major: row 64; MN-major: second chunk)
      if (a_mn) gemm_mainloop<BN, 1, 1>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, t.kb0, t.kb1, a_off, lane);
      else if (b_mn) gemm_mainloop<BN, 0, 1>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, t.kb0, t.kb1, a_off, lane);
      else gemm_mainloop<BN, 0, 0>(acc, sA, sB, full_bar, empty_bar, nstages, stage, phase, t.kb0, t.kb1, a_off, lane);
    }
    float rscale[2] = {1.f, 1.f};
    if (flags & EPI_ROW_SCALE) {
      if (in0) rscale[0] = __ldg(p.row_scale + row0 / p.rows_per_scale);
      if (in1) rscale[1] = __ldg(p.row_scale + (row0 + 8) / p.rows_per_scale);
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      // columns c*32 .. +31: f[4jj + 2h + e] = row row0 + 8h, column col0 + 8jj + cp + e (jj = 0..3)
      float* const f = acc + 16 * c;
      const int col0 = t.n0 + c * 32;
      const int part = out_f32 ? 0 : (c & 1);               // bf16: which 32-column half of the 64-column slice
      const bool s_begin = out_f32 || part == 0;
      const bool s_end = out_f32 || part == 1;
      uint8_t* const sbuf = sD + bufi * kStoreBufBytes;
      const uint32_t sb = smem_u32(sbuf);
      // operands of the epilogue are requested before the staging slice is waited for, so their latency overlaps it
      float bv[8];   // bias of column col0 + 8jj + cp + e at 2jj + e
      if (flags & EPI_BIAS) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int col = col0 + 8 * jj + cp;
          bv[2 * jj] = col < p.N ? __ldg(p.bias + col) : 0.f;
          bv[2 * jj + 1] = col < p.N ? __ldg(p.bias + col + 1) : 0.f;
        }
      }
      float2 rf[8];     // fp32 aux operand of fragment pair 2jj + h
      uint32_t rb[8];   // bf16 aux operand (bf16x2) of fragment pair 2jj + h
      const bool has_rf = (flags & EPI_RESID) != 0;
      const bool has_rb = (flags & (EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU)) != 0;
      uint32_t mbits[2] = {0u, 0u};   // mask word of each row and the chunk's 32 columns, shifted to this thread's pairs
      if ((flags & EPI_MASK_BITS) && col0 < p.N) {
        if (in0) mbits[0] = __ldg(p.mask_bits + row0 * (p.N >> 5) + (col0 >> 5)) >> cp;
        if (in1) mbits[1] = __ldg(p.mask_bits + (row0 + 8) * (p.N >> 5) + (col0 >> 5)) >> cp;
      }
      if (!aux_tma) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int col = col0 + 8 * jj + cp;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool ok = (h ? in1 : in0) && col < p.N;
            const long long off = (row0 + 8 * h) * p.ldd + col;
            if (has_rf)
              rf[2 * jj + h] = ok ? __ldg(reinterpret_cast<const float2*>(p.resid + off)) : make_float2(0.f, 0.f);
            if (has_rb)
              rb[2 * jj + h] = ok ? __ldg(reinterpret_cast<const unsigned int*>(
                                        reinterpret_cast<const __nv_bfloat16*>(p.resid_bf16) + off))
                                  : 0u;
          }
        }
      }
      if (aux_tma && s_begin) mbar_wait(&aux_bar[bufi], (aux_phase >> bufi) & 1u);   // the aux slice has landed in this staging slice
      if (s_begin && !aux_tma) {
        // the store that last read this staging slice (2*NB slices ago) must have drained it (and the stats warps too)
        if (leader) {
          tma_store_wait_read_n(NBT - 1);
          if (V::kStatsWarps) {
            mbar_wait(&sdone_bar[bufi], ((sd_phase >> bufi) & 1u) ^ 1u);
            sd_phase ^= (1u << bufi);
          }
        }
        named_bar_sync(bar_id, 256);
      }
      __syncwarp();   // ldmatrix / stmatrix are warp-collective
      if (aux_tma) {
        // each warp reads the aux fragments of its own 16 rows of the landed slice
        if (out_f32) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const uint32_t u = (uint32_t)(((2 * jj + fu) ^ fsw) << 4);
            rf[2 * jj] = *reinterpret_cast<const float2*>(sbuf + frow + u);
            rf[2 * jj + 1] = *reinterpret_cast<const float2*>(sbuf + frow + 8 * 128 + u);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 2; ++i)
            ldmatrix_x4(sb + mrow + ((uint32_t)((4 * part + 2 * i + mu) ^ sw) << 4), rb[4 * i], rb[4 * i + 1],
                        rb[4 * i + 2], rb[4 * i + 3]);
        }
      }
      // f[k]: fragment pair k/2 = 2jj + h, column 8jj + cp + (k & 1).  One loop per operation, each behind one test of
      // the (partly run-time) flags, in the order bias, ReLU, row scale, fp32 residual, bf16 aux, AXPBY, mask.
      if (flags & EPI_BIAS) {
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] += bv[2 * (k >> 2) + (k & 1)];
      }
      if (flags & EPI_RELU) {
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] = fmaxf(f[k], 0.f);
      }
      if (flags & EPI_ROW_SCALE) {
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] *= rscale[(k >> 1) & 1];
      }
      if ((flags & EPI_RESID) && (aux_tma || has_rf)) {
#pragma unroll
        for (int k = 0; k < 16; k += 2) {
          f[k] += rf[k >> 1].x;
          f[k + 1] += rf[k >> 1].y;
        }
      }
      if ((flags & (EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU)) && (aux_tma || has_rb)) {
#pragma unroll
        for (int k = 0; k < 16; k += 2) {
          const float2 ab = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rb[k >> 1]));
          if (flags & EPI_MUL_DGELU) {
            f[k] *= gelu_erf_grad(ab.x);
            f[k + 1] *= gelu_erf_grad(ab.y);
          } else if (flags & EPI_MUL_DRELU) {   // resid_bf16 = ReLU output: pass the gradient where it is > 0
            f[k] = ab.x > 0.f ? f[k] : 0.f;
            f[k + 1] = ab.y > 0.f ? f[k + 1] : 0.f;
          } else {
            f[k] += ab.x;
            f[k + 1] += ab.y;
          }
        }
      }
      if (flags & EPI_AXPBY) {
#pragma unroll
        for (int k = 0; k < 16; k += 2) {
          const float2 ab = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rb[k >> 1]));
          f[k] = fmaf(p.beta, ab.x, p.alpha * f[k]);
          f[k + 1] = fmaf(p.beta, ab.y, p.alpha * f[k + 1]);
        }
      }
      if (flags & EPI_MASK_BITS) {
        // a multiply by 0 / 1, not a select: the zeros keep the sign a later (bf16(D) * relu'(out)) would give them
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] *= ((mbits[(k >> 1) & 1] >> (8 * (k >> 2) + (k & 1))) & 1u) ? 1.f : 0.f;
      }
      if (out_f32) {
        // one 128 B (32 x fp32) slice per TMA store
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const uint32_t u = (uint32_t)(((2 * jj + fu) ^ fsw) << 4);
          *reinterpret_cast<float2*>(sbuf + frow + u) = make_float2(f[4 * jj], f[4 * jj + 1]);
          *reinterpret_cast<float2*>(sbuf + frow + 8 * 128 + u) = make_float2(f[4 * jj + 2], f[4 * jj + 3]);
        }
      } else {
        // bf16: two 32-column chunks make one 128 B (64 x bf16) slice; one x4 per 16 x 16 block
#pragma unroll
        for (int i = 0; i < 2; ++i)
          stmatrix_x4(sb + mrow + ((uint32_t)((4 * part + 2 * i + mu) ^ sw) << 4), pack_bf16x2(f[8 * i], f[8 * i + 1]),
                      pack_bf16x2(f[8 * i + 2], f[8 * i + 3]), pack_bf16x2(f[8 * i + 4], f[8 * i + 5]),
                      pack_bf16x2(f[8 * i + 6], f[8 * i + 7]));
      }
      if (s_end) {
        fence_proxy_async_smem();
        named_bar_sync(bar_id, 256);
        const int scol = out_f32 ? col0 : col0 - 32;
        if (leader) {
          if (scol < p.N && sched.phases > 1) {
            const int ab = p.ph_out[t.ph];
            asm volatile(
                "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                    reinterpret_cast<uint64_t>(tmD)),
                "r"(smem_u32(sbuf)), "r"(scol), "r"(ab & 1), "r"(0), "r"(ab >> 1), "r"(t.m0 / p.g.Q)
                : "memory");
          } else if (scol < p.N) {
            asm volatile(
                "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                    reinterpret_cast<uint64_t>(tmD)),
                "r"(smem_u32(sbuf)), "r"(scol), "r"(t.m0), "r"(V::kBatch ? t.ph : t.split)
                : "memory");
          }
          tma_store_commit();
          if (aux_tma) {
            // the slice that store s-1 read becomes the landing buffer of aux slice s + LA
            tma_store_wait_read_n(1);
            request_aux();
          }
        }
        if (V::kStatsWarps && leader) mbar_arrive(&staged_bar[bufi]);   // hand the slice to the stats warps
        aux_phase ^= (1u << bufi);
        if (++bufi == NBT) bufi = 0;
      }
    }
  }
  if (leader) tma_store_wait<0>();
  if (V::kStatsWarps) {
    named_bar_sync(3, 384);
    float* dst = p.stats_partial + (long long)blockIdx.x * 2 * p.N;
    for (int j = threadIdx.x - 128; j < 2 * p.N; j += 256) dst[j] = sStat[j];
  }
}

// Statistics warps of VAR_STATS_BF16 (warps 12..15, `wq` = warp - 12): the BatchNorm column sums of every staged slice.
// Warp wq owns columns wq*16 .. +15 of every staged 64-column slice for all 128 rows (fixed ownership and summation
// order: bit-reproducible, no atomics).  Lane l reads 8 bytes (4 columns) of row i*8 + l/4: the 8 rows of one load hit 8
// distinct swizzled 16-byte chunks, so the 256-byte request is conflict free.  The 8 row-lanes are folded by shuffles and
// lanes 0..3 add to the shared-memory accumulators they alone own.
template <int BN, int VAR>
__device__ __forceinline__ void gemm_stats_warps(const GemmParams& p, const GemmSchedule<BN, VAR>& sched, const uint8_t* sD,
                                                 float* sStat, uint64_t* staged_bar, uint64_t* sdone_bar, int wq,
                                                 int lane) {
  const int piece = lane & 3;
  const int chunk = wq * 2 + (piece >> 1);
  const int r0 = lane >> 2;
  const int soff = r0 * 128 + ((chunk ^ r0) << 4) + (piece & 1) * 8;
  const int NBT = 2 * p.store_bufs;
  int b = 0;                         // staging slice of the next output slice (the epilogue's rotation)
  uint32_t st_phase = 0u;
  named_bar_sync(3, 384);            // accumulators zeroed by the epilogue warps
  for (int w = blockIdx.x; w < sched.total; w += gridDim.x) {
    const int n0 = sched.tile(w).n0;
#pragma unroll 1
    for (int j = 0; j < BN / 64; ++j) {
      mbar_wait(&staged_bar[b], (st_phase >> b) & 1u);
      const uint8_t* const sp = sD + b * kStoreBufBytes + soff;
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
      if (lane == 0) mbar_arrive(&sdone_bar[b]);
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          sx[k] += __shfl_xor_sync(0xffffffffu, sx[k], o);
          sq[k] += __shfl_xor_sync(0xffffffffu, sq[k], o);
        }
      }
      const int gcol = n0 + j * 64 + wq * 16 + piece * 4;
      if (lane < 4 && gcol < p.N) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          sStat[gcol + k] += sx[k];
          sStat[p.N + gcol + k] += sq[k];
        }
      }
      st_phase ^= (1u << b);
      b = (b + 1 == NBT) ? 0 : b + 1;
    }
  }
  named_bar_sync(3, 384);            // all slices accumulated: the epilogue warps write the partial row
}

// The kernel carves shared memory, initialises the barriers and hands each warp its role.
template <int BN, int VAR>
__global__ void __launch_bounds__(GemmVariant<VAR>::kThreads, 1)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                  const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  using V = GemmVariant<VAR>;
  constexpr int kStages = Cfg::kStages;

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by an offset from the __shared__ symbol (not by integer arithmetic on the pointer value), so that
  // the compiler still knows every access below is to shared memory and emits 32-bit LDS / STS instead of generic ones
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int nstages = p.num_stages;
  uint8_t* sA = smem;
  uint8_t* sB = smem + nstages * (BM * BK * 2);
  uint8_t* sD = smem + nstages * Cfg::kStageBytes;
  const int NB = p.store_bufs;
  float* sStat = reinterpret_cast<float*>(sD + 2 * NB * kStoreBufBytes);  // [2][N] in VAR_STATS_BF16
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sD + 2 * NB * kStoreBufBytes + (V::kStatsWarps ? ((8 * p.N + 15) & ~15) : 0));
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* aux_bar = empty_bar + kStages;   // [2 * kMaxStoreBufs]: aux slice landed in staging slice b
  uint64_t* staged_bar = aux_bar + 2 * kMaxStoreBufs;    // [2 * kMaxStoreBufs] VAR_STATS_BF16: staging slice b is staged
  uint64_t* sdone_bar = staged_bar + 2 * kMaxStoreBufs;  // [2 * kMaxStoreBufs] the four stats warps have read slice b

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

  const GemmSchedule<BN, VAR> sched(p);
  if (warp == 0) {
    if (lane == 0) gemm_producer(&tmA, &tmB, p, sched, sA, sB, full_bar, empty_bar);
    __syncwarp();
  } else if (warp >= 4 && warp < 12) {
    gemm_consumer(&tmD, &tmR, p, sched, sA, sB, sD, sStat, full_bar, empty_bar, aux_bar, staged_bar, sdone_bar, warp - 4,
                  lane);
  } else if (V::kStatsWarps && warp >= 12) {
    gemm_stats_warps(p, sched, sD, sStat, staged_bar, sdone_bar, warp - 12, lane);
  }
}

}  // namespace saicv
