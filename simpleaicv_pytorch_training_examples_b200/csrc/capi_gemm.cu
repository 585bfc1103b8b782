// Host side of the wgmma GEMM / implicit-GEMM engine: tensor-map encoding and launches
// behind the C ABI declared in include/saicv_b200.h.
#include <cudaTypedefs.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/saicv_b200.h"
#include "gemm_sm90.cuh"
#include "host_util.h"

using namespace saicv;

namespace {

PFN_cuTensorMapEncodeTiled_v12000 g_encode_tiled = nullptr;
PFN_cuTensorMapEncodeIm2col_v12000 g_encode_im2col = nullptr;
int g_sm_count = 0;
int g_driver_version = 0;
std::once_flag g_once;
bool g_init_ok = false;

void init_driver() {
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    set_error("cuTensorMapEncodeTiled not available (no CUDA driver?)");
    return;
  }
  g_encode_tiled = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    set_error("cuTensorMapEncodeIm2col not available");
    return;
  }
  g_encode_im2col = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(fn);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { set_error("cudaGetDevice failed"); return; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { set_error("cudaGetDeviceProperties failed"); return; }
  if (prop.major != 9) {
    set_error("libsaicv_b200 requires an sm_90 (H100) device, found sm_%d%d", prop.major, prop.minor);
    return;
  }
  g_sm_count = prop.multiProcessorCount;
  cudaDriverGetVersion(&g_driver_version);
  g_init_ok = true;
}

bool ensure_init() {
  std::call_once(g_once, init_driver);
  return g_init_ok;
}

// 2-D tiled map over a row-major [rows][cols] matrix, 128B swizzle.
bool encode_2d(CUtensorMap* m, const void* ptr, CUtensorMapDataType dt, int esz, uint64_t cols,
               uint64_t rows, uint64_t row_stride_elems, uint32_t box_cols, uint32_t box_rows) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride_elems * (uint64_t)esz};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode_tiled(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(2d) failed: %d (cols=%llu rows=%llu stride=%llu box=%u,%u ptr=%p)",
              (int)r, (unsigned long long)cols, (unsigned long long)rows,
              (unsigned long long)row_stride_elems, box_cols, box_rows, ptr);
    return false;
  }
  return true;
}

// 3-D map for the output: [splits][rows][cols]
bool encode_out(CUtensorMap* m, const void* ptr, bool f32, uint64_t cols, uint64_t rows,
                uint64_t ldd, uint64_t splits, uint64_t split_stride) {
  const int esz = f32 ? 4 : 2;
  cuuint64_t dims[3] = {cols, rows, splits};
  cuuint64_t strides[2] = {ldd * esz, (splits > 1 ? split_stride : ldd * rows) * esz};
  cuuint32_t box[3] = {f32 ? 32u : 64u, 128u, 1u};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode_tiled(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                              const_cast<void*>(ptr), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(out) failed: %d (cols=%llu rows=%llu ldd=%llu splits=%llu)", (int)r,
              (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ldd,
              (unsigned long long)splits);
    return false;
  }
  return true;
}

// Store map of the phase data gradient: dx [n, 2P, 2Q, c] bf16 viewed as {c, b, q, a, n*P + p} for pixel (2p+a, 2q+b);
// the box {64, 1, Q, 1, rows} is `rows` whole pixel rows of one phase, rows*Q consecutive rows of the staging slice.
bool encode_out_phases(CUtensorMap* m, void* ptr, uint64_t c, uint64_t np, uint64_t q, uint32_t rows) {
  cuuint64_t dims[5] = {c, 2, q, 2, np};
  cuuint64_t strides[4] = {c * 2, 2 * c * 2, 2 * q * c * 2, 4 * q * c * 2};
  cuuint32_t box[5] = {64u, 1u, (cuuint32_t)q, 1u, rows};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, ptr, dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(phase out) failed: %d (c=%llu rows=%llu q=%llu box rows=%u)", (int)r,
              (unsigned long long)c, (unsigned long long)np, (unsigned long long)q, rows);
    return false;
  }
  return true;
}

// im2col map over an NHWC bf16 tensor.
bool encode_im2col(CUtensorMap* m, const void* ptr, int n, int h, int w, int c, int lc_h, int lc_w,
                   int uc_h, int uc_w, int stride, uint32_t pixels_per_col) {
  cuuint64_t dims[4] = {(uint64_t)c, (uint64_t)w, (uint64_t)h, (uint64_t)n};
  cuuint64_t strides[3] = {(uint64_t)c * 2, (uint64_t)w * c * 2, (uint64_t)h * w * c * 2};
  int lower[2] = {lc_w, lc_h};
  int upper[2] = {uc_w, uc_h};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = g_encode_im2col(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides,
                               lower, upper, 64, pixels_per_col, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed: %d (n=%d h=%d w=%d c=%d lc=%d,%d uc=%d,%d stride=%d ppc=%u)",
              (int)r, n, h, w, c, lc_h, lc_w, uc_h, uc_w, stride, pixels_per_col);
    return false;
  }
  // Same driver quirk CUTLASS works around (cute/atom/copy_traits_sm90_im2col.hpp): tensors
  // smaller than 128 KiB need bit 21 of the second descriptor word cleared on drivers <= 13.1.
  if (g_driver_version <= 13010 && (uint64_t)n * h * w * c * 2 < 131072)
    reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
  return true;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Debug / tuning override read at every launch: SAICV_GEMM_TUNE="bn:stages:store_bufs" (0 = keep the default).
void tune_override(int* bn, int* stages, int* nb) {
  const char* e = getenv("SAICV_GEMM_TUNE");
  if (!e || !*e) return;
  int a = 0, b = 0, c = 0;
  sscanf(e, "%d:%d:%d", &a, &b, &c);
  if (bn && (a == 64 || a == 128)) *bn = a;
  if (stages && b > 0) *stages = b;
  if (nb && c > 0) *nb = c;
}

// Split of the 227 KB between the operand ring (stages) and the epilogue staging slices (nb per half)
// (tests/profile_gemm_tune.py sweeps it):
//  * no aux operand: two slices per half whenever >= 3 stages remain (>= 4 for reductions of 4+ k-blocks) - a TMA store
//    is then not waited for right after it was issued;
//  * aux operand by TMA: the slices are also the landing buffers of the next aux tiles, so depth matters more than ring
//    stages while the reduction is short: <= 4 k-blocks -> 3 slices / 2+ stages, fp32 tiles of <= 16 k-blocks -> 2 slices /
//    3 stages; everything longer keeps 4 stages first.
template <int BN>
void pick_smem_split(const GemmParams& p, int stat_bytes, int* stages_out, int* nb_out) {
  using Cfg = GemmCfg<BN>;
  const int budget = kSmemBudget - stat_bytes;
  const bool has_aux = p.aux_tma != 0;
  const int kb = p.kb_per_split;
  const int min_stages = has_aux ? (kb <= 4 ? 2 : (kb <= 16 && p.out_f32) ? 3 : 4) : (kb >= 4 ? 4 : 3);
  int nb = has_aux ? 3 : 2;
  while (nb > 1 && (budget - 2 * nb * kStoreBufBytes) / Cfg::kStageBytes < min_stages) --nb;
  int stages = (budget - 2 * nb * kStoreBufBytes) / Cfg::kStageBytes;
  tune_override(nullptr, &stages, &nb);
  if (nb > kMaxStoreBufs) nb = kMaxStoreBufs;
  const int fit = (budget - 2 * nb * kStoreBufBytes) / Cfg::kStageBytes;
  if (stages > fit) stages = fit;
  if (stages > Cfg::kStages) stages = Cfg::kStages;
  *stages_out = stages;
  *nb_out = nb;
}

template <int BN, int VAR>
int launch(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& d, const CUtensorMap& r, const GemmParams& p,
           cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_sm90_kernel<BN, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_error("cudaFuncSetAttribute(smem=%d): %s", Cfg::kSmemBytes, cudaGetErrorString(e));
    attr_set = true;
  }
  const int num_m = (p.M + p.tile_rows - 1) / p.tile_rows, num_n = (p.N + BN - 1) / BN;
  const long long total = (long long)num_m * num_n * p.splits * p.phases;
  const int grid = (int)(total < g_sm_count ? total : g_sm_count);
  const int stat_bytes = (p.epi_flags & EPI_STATS) ? ((8 * p.N + 15) & ~15) : 0;
  int stages = 0, nb = 1;
  pick_smem_split<BN>(p, stat_bytes, &stages, &nb);
  if (stages < 2) return set_error("gemm_sm90_kernel<%d>: %d bytes of statistics do not fit in shared memory", BN, stat_bytes);
  const_cast<GemmParams&>(p).num_stages = stages;
  const_cast<GemmParams&>(p).store_bufs = nb;
  gemm_sm90_kernel<BN, VAR><<<grid, GemmVariant<VAR>::kThreads, Cfg::kSmemBytes, st>>>(a, b, d, r, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("gemm_sm90_kernel<%d> launch: %s", BN, cudaGetErrorString(e));
  count_launch(1);
  return 0;
}

// Tile width with the least padded columns (ties -> wider tile).  128 is the widest: each of the two consumer
// warpgroups keeps a 128 x 64 fp32 accumulator in registers next to its epilogue.
int pick_bn(int N) {
  const int cand[2] = {128, 64};
  int best = 128;
  long long best_cost = -1;
  for (int i = 0; i < 2; ++i) {
    const long long cost = (long long)((N + cand[i] - 1) / cand[i]) * cand[i];
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = cand[i]; }
  }
  tune_override(&best, nullptr, nullptr);
  return best;
}

// `aux` / `aux_f32`: the epilogue operand of the output's shape (fp32 residual or bf16 addend / mask /
// pre-activation).  When its element width equals the output's it travels by TMA (GemmParams::aux_tma).
int dispatch(int bn, const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& d, GemmParams& p,
             cudaStream_t st, const void* aux = nullptr, bool aux_f32 = false) {
  CUtensorMap r = d;
  p.aux_tma = 0;
  if (p.tile_rows == 0) p.tile_rows = BM;
  if (p.phases == 0) p.phases = 1;
  const bool both = (p.epi_flags & EPI_RESID) && (p.epi_flags & (EPI_RESID_BF16 | EPI_MUL_DGELU | EPI_MUL_DRELU));
  if (aux && !both && !(p.epi_flags & EPI_DIRECT) && p.splits == 1 && aux_f32 == (p.out_f32 != 0) && aligned16(aux) &&
      !getenv("SAICV_GEMM_NO_AUX_TMA")) {
    if (!encode_out(&r, aux, aux_f32, p.N, p.M, p.ldd, 1, 0)) return 2;
    p.aux_tma = 1;
  }
  // compile-time epilogue variant (gemm_sm90.cuh GemmVariant); SAICV_GEMM_FULL_VARIANT=1 forces the run-time one
  int var = VAR_FULL;
  if (p.a_mode == A_IM2COL_MN && (p.epi_flags || !p.out_f32 || getenv("SAICV_GEMM_FULL_VARIANT")))
    return set_error("the transposed conv weight gradient runs on the plain fp32 epilogue (VAR_PLAIN_F32) only");
  if (p.phases > 1 || p.tile_rows != BM) {
    if (p.epi_flags || p.aux_tma || p.out_f32 || p.splits != 1)
      return set_error("the phase data gradient has a plain bf16 epilogue: no epilogue flags, aux operand or split-K");
    var = VAR_PHASE_BF16;
  } else if (!getenv("SAICV_GEMM_FULL_VARIANT")) {
    if (p.aux_tma && !(p.epi_flags & ~GemmVariant<VAR_AUX>::kMask)) var = VAR_AUX;
    else if (!p.aux_tma && !p.out_f32 && !(p.epi_flags & ~GemmVariant<VAR_PLAIN_BF16>::kMask))
      var = ((p.epi_flags & EPI_STATS) && !getenv("SAICV_GEMM_INLINE_STATS")) ? VAR_STATS_BF16 : VAR_PLAIN_BF16;
    else if (!p.aux_tma && p.out_f32 && !(p.epi_flags & ~GemmVariant<VAR_PLAIN_F32>::kMask)) var = VAR_PLAIN_F32;
  }
  if ((p.epi_flags & EPI_MASK_BITS) && var != VAR_AUX)
    return set_error("EPI_MASK_BITS needs the TMA aux-operand epilogue (VAR_AUX): bf16 `add` operand, one split, no overrides");
#define SAICV_LAUNCH_BN(BN_)                                                         \
  switch (var) {                                                                     \
    case VAR_PLAIN_BF16: return launch<BN_, VAR_PLAIN_BF16>(a, b, d, r, p, st);      \
    case VAR_STATS_BF16: return launch<BN_, VAR_STATS_BF16>(a, b, d, r, p, st);      \
    case VAR_PLAIN_F32: return launch<BN_, VAR_PLAIN_F32>(a, b, d, r, p, st);        \
    case VAR_AUX: return launch<BN_, VAR_AUX>(a, b, d, r, p, st);                    \
    case VAR_PHASE_BF16: return launch<BN_, VAR_PHASE_BF16>(a, b, d, r, p, st);      \
    default: return launch<BN_, VAR_FULL>(a, b, d, r, p, st);                        \
  }
  switch (bn) {
    case 64: SAICV_LAUNCH_BN(64)
    default: SAICV_LAUNCH_BN(128)
  }
#undef SAICV_LAUNCH_BN
}

// Data gradient of a 3x3 / stride 2 / pad 1 convolution on even h, w without the zero-upsampled dy: the four output
// phases (a, b) = (h mod 2, w mod 2) are stride-1 correlations over the compact dy [n, h/2, w/2, k] (gemm_sm90.cuh,
// GemmParams::phases).  Phase a of a dimension takes dy offset 0 through tap 1 (a = 0), or offsets 0 and 1 through taps
// 2 and 0 (a = 1).  The taps of a phase are reduced in the order the stride-1 kernel reduces them over the zero-upsampled
// dy (offsets ascending, rows outer), so every sum is the same: only the blocks of exact zeros are left out.
int conv_dgrad_phases(const void* dy, const void* w, const void* add, const uint32_t* mask_bits, void* dx,
                      const saicv_conv_shape* cs, cudaStream_t st) {
  if (cs->r != 3 || cs->s != 3 || cs->pad != 1 || cs->h % 2 || cs->w % 2 || cs->w / 2 > BM)
    return set_error("saicv_conv_dgrad: stride 2 needs a 3x3 pad-1 conv on even h, w with w <= %d (r=%d s=%d pad=%d "
                     "h=%d w=%d); zero-upsample dy and pass stride 1 otherwise", 2 * BM, cs->r, cs->s, cs->pad, cs->h, cs->w);
  if (add || mask_bits) return set_error("saicv_conv_dgrad: stride 2 takes no `add` / `mask_bits`");
  const int P = cs->h / 2, Q = cs->w / 2;
  const int rows = BM / Q;   // whole dy rows per tile: the 5-D store box cannot wrap inside a row
  CUtensorMap ta, tb, td;
  if (!encode_im2col(&ta, dy, cs->n, P, Q, cs->k, 0, 0, 0, 0, 1, 128)) return 2;
  const int Kw = 9 * cs->c;
  if (!encode_2d(&tb, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, Kw, cs->k, Kw, 64, 64)) return 2;
  if (!encode_out_phases(&td, dx, cs->c, (uint64_t)cs->n * P, Q, rows)) return 2;
  GemmParams p{};
  p.M = cs->n * P * Q; p.N = cs->c; p.num_kb = 4 * (cs->k / 64); p.kb_per_split = p.num_kb; p.splits = 1;
  p.a_mode = A_IM2COL; p.b_mode = B_MN2D; p.b_cin = cs->c;
  p.g.P = P; p.g.Q = Q; p.g.stride = 1; p.g.lc_h = 0; p.g.lc_w = 0;
  p.g.R = 3; p.g.S = 3; p.g.cchunks = cs->k / 64; p.g.n_img = cs->n;
  p.epi_flags = 0; p.out_f32 = 0; p.out = dx; p.ldd = cs->c;
  p.tile_rows = rows * Q;
  p.phases = 4;
  // (weight tap, dy offset) of each output parity along one dimension
  const int taps1[2][2] = {{1, -1}, {2, 0}};
  const int order[4] = {3, 1, 2, 0};   // the 4-tap phase first, the 1-tap phase last: the short work items end the launch
  for (int i = 0; i < 4; ++i) {
    const int a = order[i] >> 1, b = order[i] & 1;
    p.ph_out[i] = order[i];
    p.ph_taps[i] = (1 + a) * (1 + b);
    int t = 0;
    for (int dr = 0; dr <= a; ++dr)
      for (int ds = 0; ds <= b; ++ds)
        p.ph_tab[i][t++] = (taps1[a][dr] * 3 + taps1[b][ds]) | (dr << 8) | (ds << 9);
  }
  return dispatch(pick_bn(cs->c), ta, tb, td, p, st);
}

}  // namespace

extern "C" {

int saicv_sm_count(void) { return ensure_init() ? g_sm_count : 0; }

int saicv_gemm_stats_rows(long long out_rows, int out_cols) {
  // number of partial rows a stats-fused forward GEMM writes = its grid size
  const int bn = pick_bn(out_cols);
  const long long tiles = ((out_rows + BM - 1) / BM) * ((out_cols + bn - 1) / bn);
  const int sms = ensure_init() ? g_sm_count : 132;
  return (int)(tiles < sms ? tiles : sms);
}

int saicv_wgrad_transposed(int out_rows, int out_cols) {
  // padded tile area of dW [rows, cols] against dW^T: few filters (rows) leave most of every 128-row tile empty
  const int bn = pick_bn(out_cols), bnt = pick_bn(out_rows);
  const long long cost = (long long)((out_rows + BM - 1) / BM) * BM * ((out_cols + bn - 1) / bn) * bn;
  const long long cost_t = (long long)((out_cols + BM - 1) / BM) * BM * ((out_rows + bnt - 1) / bnt) * bnt;
  return cost_t < cost ? 1 : 0;
}

int saicv_wgrad_splits(int out_rows, int out_cols, long long reduce_len) {
  const int bn = pick_bn(out_cols);
  const long long tiles = (long long)((out_rows + BM - 1) / BM) * ((out_cols + bn - 1) / bn);
  const long long num_kb = (reduce_len + BK - 1) / BK;
  const int sms = g_sm_count > 0 ? g_sm_count : 132;
  long long want = (2LL * sms + tiles - 1) / tiles;      // ~2 work items per SM
  long long max_by_k = num_kb / 8 > 0 ? num_kb / 8 : 1;  // at least 8 k-blocks per split
  long long s = want < max_by_k ? want : max_by_k;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  // every split must own at least one k-block
  long long per = (num_kb + s - 1) / s;
  s = (num_kb + per - 1) / per;
  return (int)s;
}

int saicv_linear_fwd(const void* x, const void* w, const float* bias, const float* resid,
                     const float* row_scale, int rows_per_scale, float* stats_partial, void* y, int M, int N,
                     int K, int flags, int out_f32, void* stream) {
  if (!ensure_init()) return 1;
  if (!aligned16(x) || !aligned16(w) || !aligned16(y) || (K % 8) || (N % (out_f32 ? 4 : 8)))
    return set_error("saicv_linear_fwd: unaligned operand (M=%d N=%d K=%d)", M, N, K);
  const int bn = pick_bn(N);
  CUtensorMap ta, tb, td;
  if (!encode_2d(&ta, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, M, K, 64, 128)) return 2;
  if (!encode_2d(&tb, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, N, K, 64, bn)) return 2;
  if (!encode_out(&td, y, out_f32, N, M, N, 1, 0)) return 2;
  GemmParams p{};
  p.M = M; p.N = N; p.num_kb = (K + BK - 1) / BK; p.kb_per_split = p.num_kb; p.splits = 1;
  p.a_mode = A_K2D; p.b_mode = B_K2D;
  p.g.P = p.g.Q = 1; p.g.cchunks = 1; p.g.S = 1; p.g.R = 1;
  p.epi_flags = (flags & (EPI_RELU | EPI_GELU | EPI_DIRECT)) | (bias ? EPI_BIAS : 0) | (resid ? EPI_RESID : 0) |
                (row_scale ? EPI_ROW_SCALE : 0);
  if (row_scale && rows_per_scale <= 0) return set_error("saicv_linear_fwd: rows_per_scale must be > 0");
  p.row_scale = row_scale; p.rows_per_scale = rows_per_scale;
  if (stats_partial) {
    if (bias || resid || out_f32 || (flags & EPI_DIRECT))
      return set_error("saicv_linear_fwd: stats_partial needs a plain bf16 output through the TMA-store epilogue (no bias / residual)");
    p.epi_flags |= EPI_STATS; p.stats_partial = stats_partial;
  }
  p.out_f32 = out_f32; p.bias = bias; p.resid = resid; p.out = y; p.ldd = N; p.split_stride = 0;
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream, resid, true);
}

int saicv_linear_dgrad(const void* dy, const void* w, const float* resid, const void* gelu_pre, void* dx,
                       int M, int N, int K, int flags, int out_f32, void* stream) {
  if (!ensure_init()) return 1;
  if (!aligned16(dy) || !aligned16(w) || !aligned16(dx) || (K % 8) || (N % 8))
    return set_error("saicv_linear_dgrad: unaligned operand (M=%d N=%d K=%d)", M, N, K);
  // GEMM: D[M, K] = dy[M, N] * W[N, K]; reduction over N; B = W stored [N(red)][K(out)] -> MN-major
  const int bn = pick_bn(K);
  CUtensorMap ta, tb, td;
  if (!encode_2d(&ta, dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, N, M, N, 64, 128)) return 2;
  if (!encode_2d(&tb, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, N, K, 64, 64)) return 2;
  if (!encode_out(&td, dx, out_f32, K, M, K, 1, 0)) return 2;
  GemmParams p{};
  p.M = M; p.N = K; p.num_kb = (N + BK - 1) / BK; p.kb_per_split = p.num_kb; p.splits = 1;
  p.a_mode = A_K2D; p.b_mode = B_MN2D;
  p.g.P = p.g.Q = 1; p.g.cchunks = 1; p.g.S = 1; p.g.R = 1;
  // aux bf16 operand [M, K]: SAICV_EPI_MUL_DRELU -> ReLU output (mask), SAICV_EPI_ADD_BF16 -> added, default -> dGELU pre-activation
  const int aux_mode = !gelu_pre ? 0 : (flags & EPI_MUL_DRELU) ? EPI_MUL_DRELU : (flags & EPI_RESID_BF16) ? EPI_RESID_BF16 : EPI_MUL_DGELU;
  p.epi_flags = (flags & EPI_DIRECT) | (resid ? EPI_RESID : 0) | aux_mode;
  if (gelu_pre && !aligned16(gelu_pre)) return set_error("saicv_linear_dgrad: unaligned aux operand");
  p.out_f32 = out_f32; p.resid = resid; p.resid_bf16 = gelu_pre; p.out = dx; p.ldd = K;
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream, resid ? (const void*)resid : gelu_pre, resid != nullptr);
}

int saicv_linear_wgrad(const void* dy, const void* x, float* dw_partial, int M, int N, int K,
                       int splits, void* stream) {
  if (!ensure_init()) return 1;
  if (!aligned16(dy) || !aligned16(x) || !aligned16(dw_partial) || (K % 8) || (N % 8))
    return set_error("saicv_linear_wgrad: unaligned operand (M=%d N=%d K=%d)", M, N, K);
  // GEMM: D[N, K] = dy[M, N]^T * x[M, K]; reduction over M; both operands MN-major
  const int bn = pick_bn(K);
  CUtensorMap ta, tb, td;
  if (!encode_2d(&ta, dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, N, M, N, 64, 64)) return 2;
  if (!encode_2d(&tb, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, M, K, 64, 64)) return 2;
  if (!encode_out(&td, dw_partial, true, K, N, K, splits, (uint64_t)N * K)) return 2;
  GemmParams p{};
  p.M = N; p.N = K; p.num_kb = (M + BK - 1) / BK;
  p.kb_per_split = (p.num_kb + splits - 1) / splits;
  p.splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;
  if (p.splits != splits) return set_error("saicv_linear_wgrad: splits=%d leaves an empty split (use saicv_wgrad_splits)", splits);
  p.a_mode = A_MN2D; p.b_mode = B_MN2D;
  p.g.P = p.g.Q = 1; p.g.cchunks = 1; p.g.S = 1; p.g.R = 1;
  p.epi_flags = 0; p.out_f32 = 1; p.out = dw_partial; p.ldd = K; p.split_stride = (long long)N * K;
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream);
}

static int conv_out(int in, int pad, int r, int stride) { return (in + 2 * pad - r) / stride + 1; }

int saicv_conv_fprop(const void* x, const void* w, float* stats_partial, void* y, const saicv_conv_shape* cs,
                     int flags, void* stream) {
  if (!ensure_init()) return 1;
  if (cs->c % 64 || cs->k % 8 || !aligned16(x) || !aligned16(w) || !aligned16(y))
    return set_error("saicv_conv_fprop: needs c%%64==0, k%%8==0 and 16B-aligned pointers (c=%d k=%d)", cs->c, cs->k);
  const int P = conv_out(cs->h, cs->pad, cs->r, cs->stride), Q = conv_out(cs->w, cs->pad, cs->s, cs->stride);
  const long long M = (long long)cs->n * P * Q;
  const int Kred = cs->r * cs->s * cs->c;
  const int bn = pick_bn(cs->k);
  CUtensorMap ta, tb, td;
  if (!encode_im2col(&ta, x, cs->n, cs->h, cs->w, cs->c, -cs->pad, -cs->pad, cs->pad - (cs->r - 1),
                     cs->pad - (cs->s - 1), cs->stride, 128))
    return 2;
  if (!encode_2d(&tb, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, Kred, cs->k, Kred, 64, bn)) return 2;
  if (!encode_out(&td, y, false, cs->k, M, cs->k, 1, 0)) return 2;
  GemmParams p{};
  p.M = (int)M; p.N = cs->k; p.num_kb = Kred / BK; p.kb_per_split = p.num_kb; p.splits = 1;
  p.a_mode = A_IM2COL; p.b_mode = B_K2D; p.b_cin = cs->c;
  p.g.P = P; p.g.Q = Q; p.g.stride = cs->stride; p.g.lc_h = -cs->pad; p.g.lc_w = -cs->pad;
  p.g.R = cs->r; p.g.S = cs->s; p.g.cchunks = cs->c / 64; p.g.n_img = cs->n;
  p.epi_flags = flags & (EPI_RELU | EPI_DIRECT); p.out_f32 = 0; p.out = y; p.ldd = cs->k;
  if (stats_partial) {
    if (flags & EPI_DIRECT) return set_error("saicv_conv_fprop: stats_partial is not available with SAICV_EPI_DIRECT");
    p.epi_flags |= EPI_STATS; p.stats_partial = stats_partial;
  }
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream);
}

int saicv_conv_dgrad(const void* dy, const void* w, const void* add, const uint32_t* mask_bits, void* dx,
                     const saicv_conv_shape* cs, void* stream) {
  if (!ensure_init()) return 1;
  if (cs->c % 64 || cs->k % 64 || !aligned16(dy) || !aligned16(w) || !aligned16(dx))
    return set_error("saicv_conv_dgrad: needs c%%64==0 and k%%64==0 (c=%d k=%d)", cs->c, cs->k);
  if (cs->stride == 2) return conv_dgrad_phases(dy, w, add, mask_bits, dx, cs, (cudaStream_t)stream);
  if (cs->stride != 1)
    return set_error("saicv_conv_dgrad: stride %d (1, or 2 for 3x3 pad 1 on even sizes)", cs->stride);
  // dy has spatial extent (h, w) and k channels; output dx [n,h,w,c].
  const long long M = (long long)cs->n * cs->h * cs->w;
  const int Kw = cs->r * cs->s * cs->c;  // weight row length
  const int bn = pick_bn(cs->c);
  const int lc_h = cs->pad - (cs->r - 1), lc_w = cs->pad - (cs->s - 1);
  CUtensorMap ta, tb, td;
  if (!encode_im2col(&ta, dy, cs->n, cs->h, cs->w, cs->k, lc_h, lc_w, lc_h, lc_w, 1, 128)) return 2;
  if (!encode_2d(&tb, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, Kw, cs->k, Kw, 64, 64)) return 2;
  if (!encode_out(&td, dx, false, cs->c, M, cs->c, 1, 0)) return 2;
  GemmParams p{};
  p.M = (int)M; p.N = cs->c; p.num_kb = cs->r * cs->s * (cs->k / 64); p.kb_per_split = p.num_kb; p.splits = 1;
  p.a_mode = A_IM2COL; p.b_mode = B_MN2D; p.flip_taps = 1; p.b_cin = cs->c;
  p.g.P = cs->h; p.g.Q = cs->w; p.g.stride = 1; p.g.lc_h = lc_h; p.g.lc_w = lc_w;
  p.g.R = cs->r; p.g.S = cs->s; p.g.cchunks = cs->k / 64; p.g.n_img = cs->n;
  p.epi_flags = (add ? EPI_RESID_BF16 : 0) | (mask_bits ? EPI_MASK_BITS : 0);
  p.resid_bf16 = add; p.mask_bits = mask_bits; p.out_f32 = 0; p.out = dx; p.ldd = cs->c;
  if (add && !aligned16(add)) return set_error("saicv_conv_dgrad: unaligned `add`");
  if (mask_bits && !add) return set_error("saicv_conv_dgrad: mask_bits is applied in the epilogue of the fused `add` only");
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream, add, false);
}

int saicv_conv_wgrad(const void* dy, const void* x, float* dw_partial, const saicv_conv_shape* cs,
                     int splits, void* stream) {
  if (!ensure_init()) return 1;
  if (cs->c % 64 || cs->k % 8 || !aligned16(dy) || !aligned16(x) || !aligned16(dw_partial))
    return set_error("saicv_conv_wgrad: needs c%%64==0, k%%8==0 (c=%d k=%d)", cs->c, cs->k);
  const int P = conv_out(cs->h, cs->pad, cs->r, cs->stride), Q = conv_out(cs->w, cs->pad, cs->s, cs->stride);
  const long long Mpix = (long long)cs->n * P * Q;
  const int Ncols = cs->r * cs->s * cs->c;
  // splits: saicv_wgrad_splits in the dW orientation, whichever product runs, so that both reduce the same k-blocks
  const bool tr = saicv_wgrad_transposed(cs->k, Ncols) != 0;
  const int bn = pick_bn(tr ? cs->k : Ncols);
  CUtensorMap ta, tb, td;
  CUtensorMap& tdy = tr ? tb : ta;
  CUtensorMap& tx = tr ? ta : tb;
  if (!encode_2d(&tdy, dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, cs->k, Mpix, cs->k, 64, 64)) return 2;
  if (!encode_im2col(&tx, x, cs->n, cs->h, cs->w, cs->c, -cs->pad, -cs->pad, cs->pad - (cs->r - 1),
                     cs->pad - (cs->s - 1), cs->stride, 64))
    return 2;
  if (tr ? !encode_out(&td, dw_partial, true, cs->k, Ncols, cs->k, splits, (uint64_t)cs->k * Ncols)
         : !encode_out(&td, dw_partial, true, Ncols, cs->k, Ncols, splits, (uint64_t)cs->k * Ncols))
    return 2;
  GemmParams p{};
  p.M = tr ? Ncols : cs->k; p.N = tr ? cs->k : Ncols; p.num_kb = (int)((Mpix + BK - 1) / BK);
  p.kb_per_split = (p.num_kb + splits - 1) / splits;
  p.splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;
  if (p.splits != splits) return set_error("saicv_conv_wgrad: splits=%d leaves an empty split (use saicv_wgrad_splits)", splits);
  p.a_mode = tr ? A_IM2COL_MN : A_MN2D; p.b_mode = tr ? B_MN2D : B_IM2COL;
  p.g.P = P; p.g.Q = Q; p.g.stride = cs->stride; p.g.lc_h = -cs->pad; p.g.lc_w = -cs->pad;
  p.g.R = cs->r; p.g.S = cs->s; p.g.cchunks = cs->c / 64; p.g.n_img = cs->n;
  p.epi_flags = 0; p.out_f32 = 1; p.out = dw_partial; p.ldd = p.N; p.split_stride = (long long)cs->k * Ncols;
  return dispatch(bn, ta, tb, td, p, (cudaStream_t)stream);
}

}  // extern "C"
