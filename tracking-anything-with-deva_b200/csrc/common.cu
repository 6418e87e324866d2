#include "common.h"

#include <stdarg.h>

namespace b200 {

static thread_local char g_error[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_error; }

static unsigned long long g_launches = 0;
void count_launch() { __atomic_add_fetch(&g_launches, 1ull, __ATOMIC_RELAXED); }
unsigned long long launch_count() { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

int sm_count() {
  static int cached[kMaxDevices] = {0};
  const int dev = device_slot();
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached[dev] = n;
    else
      cached[dev] = 132;  // H100 SXM
  }
  return cached[dev];
}

}  // namespace b200
