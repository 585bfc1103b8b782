// Host runtime shared by the translation units of libsaicv_b200.so (host_util.cu): error reporting, launch counting,
// the device query, 1-D grid sizing, and the launchers of the fold kernels that more than one unit reduces through.
#pragma once
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

namespace saicv {
// Formats into a thread-local buffer returned by saicv_last_error(); always returns 1.
int set_error(const char* fmt, ...);
int check_launch(const char* what);
// Number of kernels this library has launched in this process (bench.py's gpu_launches).
void count_launch(int n);

// The driver entry points and properties of the current device, queried once per process.
struct Device {
  PFN_cuTensorMapEncodeTiled_v12000 encode_tiled;
  PFN_cuTensorMapEncodeIm2col_v12000 encode_im2col;
  int sms;
  int driver_version;
};
// nullptr, with saicv_last_error() set, when there is no CUDA driver or the device is not sm_90.
const Device* device();

// Default block cap of the 1-D grids: 16 blocks on each of the 132 SMs of an H100 SXM.  Grid caps are fixed counts, not
// sized from the live SM count: a reduction that writes one partial row per block folds in an order set by its grid.
constexpr int kGridCap = 132 * 16;
// ceil(items / per_block) blocks, clamped to [1, cap].
int grid_1d(long long items, int per_block = 256, int cap = kGridCap);
// The least power of two >= v.
int pow2_ge(int v);

// Fixed-order fold of nblk partial rows [nblk][ncols]: out0[j] (+)= sum_b partials[b][j] for j < split, and
// out1[j - split] for split <= j < ncols.  One launch of (ncols + 7) / 8 blocks (capi_elementwise.cu).
int fold_partials(const float* partials, int nblk, int ncols, float* out0, float* out1, int split, int accumulate,
                  cudaStream_t st);
// BatchNorm parameter gradients from the reduced sums [2][c] (sum g | sum g * xhat): dbeta (+)= sums[0 .. c),
// dgamma (+)= sums[c .. 2c) (capi_elementwise.cu).
int bn_param_grad(const float* sums, float* dgamma, float* dbeta, int c, int accumulate, cudaStream_t st);

// The row count of a cross-rank BatchNorm exchange rides in the exchanged fp32 buffer as two values, hi = rows >> 12
// and lo = rows & 4095, so that their sums over ranks stay exact integers: up to 2^36 rows over up to 4096 ranks
// (a single fp32 count is exact only up to 2^24 rows).
constexpr int kBnCountShift = 12;
__host__ __device__ inline long long bn_sync_count(const float* cnt) {
  return ((long long)cnt[0] << kBnCountShift) + (long long)cnt[1];
}
}  // namespace saicv
