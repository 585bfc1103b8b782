// Host side of the wgmma attention family (attn_sm90.cuh): tensor maps, template dispatch, launches.
#include <cudaTypedefs.h>

#include <mutex>

#include "../../include/saicv_b200.h"
#include "attn_sm90.cuh"
#include "host_util.h"

using namespace saicv;

namespace {

PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
int g_sms = 0;
std::once_flag g_once;
bool g_ok = false;

void init() {
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    set_error("cuTensorMapEncodeTiled not available (no CUDA driver?)");
    return;
  }
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    set_error("cudaGetDeviceProperties failed");
    return;
  }
  if (prop.major != 9) {
    set_error("libsaicv_b200 requires an sm_90 (H100) device, found sm_%d%d", prop.major, prop.minor);
    return;
  }
  g_sms = prop.multiProcessorCount;
  g_ok = true;
}
bool ensure() {
  std::call_once(g_once, init);
  return g_ok;
}

// [B][H][L][D] view with arbitrary (16-byte aligned) strides; box = 64 columns x `rows` rows, 128B swizzle,
// out-of-range rows / columns read as zero.
bool encode_4d(CUtensorMap* m, const void* ptr, int D, int L, int H, int B, const long long* strides /*b,h,row*/,
               uint32_t rows) {
  cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)L, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t st[3] = {(cuuint64_t)strides[2] * 2, (cuuint64_t)strides[1] * 2, (cuuint64_t)strides[0] * 2};
  cuuint32_t box[4] = {64, rows, 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (st[0] & 15) || (st[1] & 15) || (st[2] & 15)) {
    set_error("attention operand not 16-byte aligned (ptr %p strides %lld %lld %lld elements)", ptr, strides[0], strides[1], strides[2]);
    return false;
  }
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, st, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(attention 4d) failed: %d (D=%d L=%d H=%d B=%d strides %lld %lld %lld)", (int)r, D, L, H, B,
              strides[0], strides[1], strides[2]);
    return false;
  }
  return true;
}

// persistent grid: MINB (1 or 2) CTAs per SM; the kernels are compiled with __launch_bounds__(160, MINB) and
// their shared-memory footprints are sized for exactly that residency
template <typename K>
int persistent_grid(K kernel, int minb, long long total) {
  static bool carve = false;
  if (!carve) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    carve = true;
  }
  const long long g = (long long)g_sms * minb;
  return (int)(total < g ? total : g);
}

AttnDrop make_drop(const saicv_attn_args* a) {
  AttnDrop d{};
  if (a->dropout_p > 0.f) {
    d.thresh = dropout_threshold(a->dropout_p);
    d.seed_lo = (uint32_t)a->dropout_seed;
    d.seed_hi = (uint32_t)(a->dropout_seed >> 32);
    d.scale = 1.f / (1.f - a->dropout_p);
    d.seed_base = a->dropout_seed_base;
  }
  return d;
}

template <int DQK, int DV, int MINB, bool DROP>
int launch_fwd(const saicv_attn_args* a, cudaStream_t st) {
  using Cfg = AttnFwdCfg<DQK, DV>;
  auto kernel = attn_fwd_sm90_kernel<DQK, DV, MINB, DROP>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return set_error("attention fwd<%d,%d>: smem %d: %s", DQK, DV, Cfg::kSmemBytes, cudaGetErrorString(e));
    }
    attr = true;
  }
  CUtensorMap tq, tk, tv;
  if (!encode_4d(&tq, a->q, DQK, a->lq, a->h, a->b, a->q_strides, kAttnRows)) return 2;
  if (!encode_4d(&tk, a->k, DQK, a->lk, a->h, a->b, a->k_strides, kAttnCols)) return 2;
  if (!encode_4d(&tv, a->v, DV, a->lk, a->h, a->b, a->v_strides, kAttnCols)) return 2;
  AttnParams p{};
  p.B = a->b; p.H = a->h; p.Lq = a->lq; p.Lk = a->lk;
  p.num_q_tiles = (a->lq + kAttnRows - 1) / kAttnRows;
  p.scale = a->scale;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out);
  p.o_sb = a->o_strides[0]; p.o_sh = a->o_strides[1]; p.o_sl = a->o_strides[2];
  p.lse = a->lse;
  p.mask_bits = a->key_mask_bits; p.mask_words = a->mask_words;
  p.drop = make_drop(a);
  const long long total = (long long)a->b * a->h * p.num_q_tiles;
  const int grid = persistent_grid(kernel, MINB, total);
  kernel<<<grid, kAttnThreads, Cfg::kSmemBytes, st>>>(tq, tk, tv, p);
  return check_launch("attn_fwd_sm90_kernel");
}

template <int DQK, int DV, bool KEYS, int MINB, bool DROP>
int launch_bwd_phase(const saicv_attn_bwd_args* a, cudaStream_t st) {
  using Cfg = AttnBwdCfg<DQK, DV, KEYS>;
  auto kernel = attn_bwd_sm90_kernel<DQK, DV, KEYS, MINB, DROP>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return set_error("attention bwd<%d,%d,%d>: smem %d: %s", DQK, DV, (int)KEYS, Cfg::kSmemBytes, cudaGetErrorString(e));
    }
    attr = true;
  }
  const saicv_attn_args* f = &a->fwd;
  CUtensorMap r0, r1, c0, c1;
  if (!KEYS) {
    if (!encode_4d(&r0, f->q, DQK, f->lq, f->h, f->b, f->q_strides, kAttnRows)) return 2;
    if (!encode_4d(&r1, a->dout, DV, f->lq, f->h, f->b, f->o_strides, kAttnRows)) return 2;
    if (!encode_4d(&c0, f->k, DQK, f->lk, f->h, f->b, f->k_strides, kAttnCols)) return 2;
    if (!encode_4d(&c1, f->v, DV, f->lk, f->h, f->b, f->v_strides, kAttnCols)) return 2;
  } else {
    if (!encode_4d(&r0, f->k, DQK, f->lk, f->h, f->b, f->k_strides, kAttnRows)) return 2;
    if (!encode_4d(&r1, f->v, DV, f->lk, f->h, f->b, f->v_strides, kAttnRows)) return 2;
    if (!encode_4d(&c0, f->q, DQK, f->lq, f->h, f->b, f->q_strides, kAttnCols)) return 2;
    if (!encode_4d(&c1, a->dout, DV, f->lq, f->h, f->b, f->o_strides, kAttnCols)) return 2;
  }
  AttnBwdParams p{};
  p.B = f->b; p.H = f->h; p.Lq = f->lq; p.Lk = f->lk;
  p.num_tiles = ((KEYS ? f->lk : f->lq) + kAttnRows - 1) / kAttnRows;
  p.scale = f->scale;
  p.scale_log2 = f->scale * 1.4426950408889634f;
  p.lse = f->lse; p.delta = a->delta;
  p.mask_bits = f->key_mask_bits; p.mask_words = f->mask_words;
  p.drop = make_drop(f);
  if (!KEYS) {
    p.d_out0 = reinterpret_cast<__nv_bfloat16*>(a->dq);
    p.s0b = a->dq_strides[0]; p.s0h = a->dq_strides[1]; p.s0l = a->dq_strides[2];
  } else {
    p.d_out0 = reinterpret_cast<__nv_bfloat16*>(a->dk);
    p.s0b = a->dk_strides[0]; p.s0h = a->dk_strides[1]; p.s0l = a->dk_strides[2];
    p.d_out1 = reinterpret_cast<__nv_bfloat16*>(a->dv);
    p.s1b = a->dv_strides[0]; p.s1h = a->dv_strides[1]; p.s1l = a->dv_strides[2];
  }
  p.dk_cols = a->dk_cols > 0 ? a->dk_cols : DQK;
  const long long total = (long long)f->b * f->h * p.num_tiles;
  const int grid = persistent_grid(kernel, MINB, total);
  kernel<<<grid, kAttnThreads, Cfg::kSmemBytes, st>>>(r0, r1, c0, c1, p);
  return check_launch("attn_bwd_sm90_kernel");
}

// delta[b][h][q] = sum_d dO * O.  Each thread reads 16-byte pieces (8 bf16) of both rows; a row of DV values is shared
// by DV / 8 adjacent lanes (8 for hd 64, 10 for hd 80, 4 for hd 32) and folded with shuffles inside groups of 16 lanes.
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o, float* __restrict__ delta,
                                  int B, int H, int L, int DV, long long sb, long long sh, long long sl) {
  const long long rows = (long long)B * H * L;
  const int sub = threadIdx.x & 15;                      // lane inside the 16-lane group that owns one row
  const int pieces = DV >> 3;                            // <= 16 (DV <= 128)
  const long long groups = ((long long)gridDim.x * blockDim.x) >> 4;
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4; r < rows; r += groups) {
    const int q = (int)(r % L);
    const long long bh = r / L;
    const int h = (int)(bh % H);
    const long long b = bh / H;
    const long long off = b * sb + h * sh + q * sl;
    float s = 0.f;
    if (sub < pieces) {
      const uint4 x = __ldg(reinterpret_cast<const uint4*>(o + off) + sub);
      const uint4 y = __ldg(reinterpret_cast<const uint4*>(d_o + off) + sub);
      const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int k = 0; k < 4; ++k)
        s += __uint_as_float(xw[k] << 16) * __uint_as_float(yw[k] << 16) +
             __uint_as_float(xw[k] & 0xffff0000u) * __uint_as_float(yw[k] & 0xffff0000u);
    }
#pragma unroll
    for (int m = 8; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if (sub == 0) delta[r] = s;
  }
}

template <int DQK, int DV>
constexpr bool kDropoutShape = (DQK == 32 && DV == 32) || (DQK == 48 && DV == 32) || (DQK == 64 && DV == 64);

template <int DQK, int DV>
int fwd_for(const saicv_attn_args* a, cudaStream_t st) {
  // two CTAs per SM whenever the tiles of both fit
  constexpr bool two = AttnFwdCfg<DQK, DV>::kSmemBytes <= 115712;
  if (a->dropout_p > 0.f) {
    // attention-probability dropout is compiled for the head sizes that train with it (DETR hd 32 with / without the
    // key-bias column, ViT hd 64); the other shapes keep the mask-free instruction stream only
    if constexpr (kDropoutShape<DQK, DV>) return launch_fwd<DQK, DV, two ? 2 : 1, true>(a, st);
    else return set_error("attention dropout is not compiled for (score width, value width) = (%d, %d)", DQK, DV);
  }
  return launch_fwd<DQK, DV, two ? 2 : 1, false>(a, st);
}
template <int DQK, int DV>
int bwd_for(const saicv_attn_bwd_args* a, cudaStream_t st) {
  // two CTAs per SM (<= 204 registers a thread) while the accumulators stay small: S, dP (32 + 32) + dQ or dV + dK
  constexpr bool twoA = 64 + DQK / 2 <= 128 && AttnBwdCfg<DQK, DV, false>::kSmemBytes <= 115712;
  constexpr bool twoB = 64 + DV / 2 + DQK / 2 <= 128 && AttnBwdCfg<DQK, DV, true>::kSmemBytes <= 115712;
  if (a->fwd.dropout_p > 0.f) {
    if constexpr (kDropoutShape<DQK, DV>) {
      if (int e = launch_bwd_phase<DQK, DV, false, twoA ? 2 : 1, true>(a, st)) return e;
      return launch_bwd_phase<DQK, DV, true, twoB ? 2 : 1, true>(a, st);
    } else {
      return set_error("attention dropout is not compiled for (score width, value width) = (%d, %d)", DQK, DV);
    }
  }
  if (int e = launch_bwd_phase<DQK, DV, false, twoA ? 2 : 1, false>(a, st)) return e;
  return launch_bwd_phase<DQK, DV, true, twoB ? 2 : 1, false>(a, st);
}

#define SAICV_ATTN_SHAPES(X) X(32, 32) X(48, 32) X(64, 64) X(80, 80) X(96, 64) X(112, 64) X(112, 80) X(128, 80) X(192, 64) X(208, 80)

}  // namespace

extern "C" {

int saicv_attn_fwd(const saicv_attn_args* a, void* stream) {
  if (!ensure()) return 1;
  if (a->lq < 1 || a->lk < 1 || a->b < 1 || a->h < 1) return set_error("saicv_attn_fwd: empty problem");
  if (!(a->scale > 0.f)) return set_error("saicv_attn_fwd: the softmax scale must be positive");
  if (!(a->dropout_p >= 0.f && a->dropout_p < 1.f)) return set_error("saicv_attn_fwd: dropout_p must be in [0, 1)");
  if (a->key_mask_bits && a->mask_words * 32 < ((a->lk + 127) / 128) * 128)
    return set_error("saicv_attn_fwd: mask_words must cover lk rounded up to 128 keys");
#define X(Q, V) if (a->dqk == Q && a->dv == V) return fwd_for<Q, V>(a, (cudaStream_t)stream);
  SAICV_ATTN_SHAPES(X)
#undef X
  return set_error("saicv_attn_fwd: unsupported (score width, value width) = (%d, %d)", a->dqk, a->dv);
}

int saicv_attn_bwd(const saicv_attn_bwd_args* a, void* stream) {
  if (!ensure()) return 1;
  const saicv_attn_args* f = &a->fwd;
  if (a->dk_cols < 0 || a->dk_cols > f->dqk || (a->dk_cols % 16)) return set_error("saicv_attn_bwd: bad dk_cols %d", a->dk_cols);
  {
    const long long rows = (long long)f->b * f->h * f->lq;
    if (f->dv % 8 || f->dv > 128) return set_error("saicv_attn_bwd: the value width must be a multiple of 8, <= 128 (got %d)", f->dv);
    long long blocks = (rows + 15) / 16;               // 16 rows per 256-thread block
    if (blocks > (long long)g_sms * 16) blocks = (long long)g_sms * 16;
    attn_delta_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(f->out), reinterpret_cast<const __nv_bfloat16*>(a->dout), a->delta, f->b, f->h,
        f->lq, f->dv, f->o_strides[0], f->o_strides[1], f->o_strides[2]);
    if (int e = check_launch("attn_delta_kernel")) return e;
  }
#define X(Q, V) if (f->dqk == Q && f->dv == V) return bwd_for<Q, V>(a, (cudaStream_t)stream);
  SAICV_ATTN_SHAPES(X)
#undef X
  return set_error("saicv_attn_bwd: unsupported (score width, value width) = (%d, %d)", f->dqk, f->dv);
}

// ---- packed-qkv convenience entries used by the ViT runtime: qkv [B, L, 3, H, d], out [B, L, H*d]
static void fill_packed(saicv_attn_args* a, const void* qkv, void* out, float* lse, int b, int l, int h, int d, float scale) {
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(qkv);
  const long long sl = 3LL * h * d, sb = (long long)l * sl;
  a->q = base; a->k = base + (long long)h * d; a->v = base + 2LL * h * d;
  a->out = out; a->lse = lse;
  for (auto* s : {a->q_strides, a->k_strides, a->v_strides}) { s[0] = sb; s[1] = d; s[2] = sl; }
  a->o_strides[0] = (long long)l * h * d; a->o_strides[1] = d; a->o_strides[2] = (long long)h * d;
  a->key_mask_bits = nullptr; a->mask_words = 0;
  a->b = b; a->h = h; a->lq = l; a->lk = l; a->dqk = d; a->dv = d; a->scale = scale;
}

int saicv_attention_fwd(const void* qkv, void* out, float* lse, int b, int l, int h, int d, float scale, void* stream) {
  saicv_attn_args a{};
  fill_packed(&a, qkv, out, lse, b, l, h, d, scale);
  return saicv_attn_fwd(&a, stream);
}

int saicv_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv, int b,
                        int l, int h, int d, float scale, void* stream) {
  saicv_attn_bwd_args a{};
  fill_packed(&a.fwd, qkv, const_cast<void*>(out), const_cast<float*>(lse), b, l, h, d, scale);
  a.dout = dout; a.delta = delta;
  __nv_bfloat16* g = reinterpret_cast<__nv_bfloat16*>(dqkv);
  a.dq = g; a.dk = g + (long long)h * d; a.dv = g + 2LL * h * d;
  for (auto* s : {a.dq_strides, a.dk_strides, a.dv_strides}) { s[0] = a.fwd.q_strides[0]; s[1] = d; s[2] = a.fwd.q_strides[2]; }
  a.dk_cols = d;
  return saicv_attn_bwd(&a, stream);
}

}  // extern "C"
