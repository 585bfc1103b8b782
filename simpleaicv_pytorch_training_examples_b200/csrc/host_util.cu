// Host runtime of libsaicv_b200.so: the error and launch-count state behind saicv_last_error / saicv_launch_count, the
// once-only device query the GEMM and attention engines encode their tensor maps and size their grids with, and the
// 1-D grid sizing of the streaming kernels.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>

#include "../../include/saicv_b200.h"
#include "host_util.h"

namespace saicv {
namespace {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

// Fills `d`, or writes into `why` why the device cannot run this library.
void query_device(Device* d, char* why, size_t n) {
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    snprintf(why, n, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
    return;
  }
  d->encode_tiled = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    snprintf(why, n, "cuTensorMapEncodeIm2col not available");
    return;
  }
  d->encode_im2col = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(fn);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    snprintf(why, n, "cudaGetDevice failed");
    return;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    snprintf(why, n, "cudaGetDeviceProperties failed");
    return;
  }
  if (prop.major != 9) {
    snprintf(why, n, "libsaicv_b200 requires an sm_90 (H100) device, found sm_%d%d", prop.major, prop.minor);
    return;
  }
  d->sms = prop.multiProcessorCount;
  cudaDriverGetVersion(&d->driver_version);
}

}  // namespace

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s: %s", what, cudaGetErrorString(e));
  count_launch(1);
  return 0;
}

const Device* device() {
  static Device d{};
  static char why[256] = "";
  static std::once_flag once;
  std::call_once(once, [] { query_device(&d, why, sizeof(why)); });
  // the reason is kept so that every failing call reports it, on whichever thread makes the call
  if (why[0]) {
    set_error("%s", why);
    return nullptr;
  }
  return &d;
}

int grid_1d(long long items, int per_block, int cap) {
  long long b = (items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}
int pow2_ge(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

}  // namespace saicv

extern "C" {

long long saicv_launch_count(void) { return saicv::g_launches.load(std::memory_order_relaxed); }
const char* saicv_last_error(void) { return saicv::g_err; }
int saicv_sm_count(void) {
  const saicv::Device* d = saicv::device();
  return d ? d->sms : 0;
}

}  // extern "C"
