// lib.cu -- library-level state of libsparsebit_b200.so: error string, SM count, launch counter.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace sb200 {

static thread_local char t_err[512] = "";
std::atomic<long long> g_launches{0};
int g_variant = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  // Cached per device ordinal (up to 64 devices per process).
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v > 0) return v;
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  cache[dev].store(n, std::memory_order_relaxed);
  return n;
}

}  // namespace sb200

extern "C" {

const char* sb200_last_error(void) { return sb200::t_err; }
int sb200_version(void) { return 100; }
int sb200_sm_count(void) { return sb200::sm_count(); }
int sb200_set_variant(int variant) {
  if (variant < 0 || variant > 2) {
    sb200::set_error("sb200_set_variant: variant must be 0, 1 or 2 (got %d)", variant);
    return SB200_E_INVALID;
  }
  sb200::g_variant = variant;
  return SB200_OK;
}
int64_t sb200_launch_count(void) { return (int64_t)sb200::g_launches.load(); }

}  // extern "C"
