// C-ABI plumbing: error text, launch counter, driver entry points.
#include "host.h"
#include <atomic>
#include <mutex>
#include <string.h>

namespace b200 {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 148;
  }
  return cached[dev];
}

static void* driver_entry(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess) {
    return nullptr;
  }
  return fn;
}
EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = (EncodeTiledFn)driver_entry("cuTensorMapEncodeTiled");
  return fn;
}
EncodeIm2colFn encode_im2col_fn() {
  static EncodeIm2colFn fn = (EncodeIm2colFn)driver_entry("cuTensorMapEncodeIm2col");
  return fn;
}

int wgrad_reduce_warps(int splits) {
  int w = 8;
  while (w > 1 && w > splits) w >>= 1;   // no idle warps when there are only a few splits
  return w;
}

}  // namespace b200

extern "C" {
const char* b200_last_error(void) { return b200::g_err; }
int b200_version(void) { return 100; }
long long b200_launch_count(void) { return b200::g_launches.load(); }
}
