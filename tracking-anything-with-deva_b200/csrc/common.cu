#include "common.h"

#include <stdarg.h>
#include <string.h>

namespace b200 {

static thread_local char g_error[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

static unsigned long long g_launches = 0;
void count_launch() { __atomic_add_fetch(&g_launches, 1ull, __ATOMIC_RELAXED); }

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

namespace {
struct DeviceScope {
  int prev = 0;
  explicit DeviceScope(int d) { cudaGetDevice(&prev); cudaSetDevice(d); }
  ~DeviceScope() { cudaSetDevice(prev); }
};
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API int deva_b200_abi_version(void) { return DEVA_B200_ABI_VERSION; }
DEVA_B200_API const char* deva_b200_last_error(void) { return g_error; }
DEVA_B200_API uint64_t deva_b200_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

DEVA_B200_API int deva_b200_device_check(void) {
  int dev = 0, major = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  int minor = 0;
  B200_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  B200_REQUIRE(major == 9 && minor == 0, "deva_b200 kernels are built for sm_90a; device has compute capability %d.%d", major, minor);
  return 0;
}

DEVA_B200_API int deva_b200_peer_alloc(int device, int64_t bytes, void** ptr, uint8_t handle[64]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  B200_REQUIRE(bytes > 0 && ptr && handle, "peer_alloc: bad arguments");
  DeviceScope scope(device);
  B200_CUDA(cudaMalloc(ptr, (size_t)bytes));
  B200_CUDA(cudaMemset(*ptr, 0, (size_t)bytes));
  cudaIpcMemHandle_t h;
  B200_CUDA(cudaIpcGetMemHandle(&h, *ptr));
  memcpy(handle, &h, 64);
  return 0;
}
DEVA_B200_API int deva_b200_peer_open(int device, const uint8_t handle[64], void** ptr) {
  B200_REQUIRE(ptr && handle, "peer_open: bad arguments");
  DeviceScope scope(device);
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  B200_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
DEVA_B200_API int deva_b200_peer_close(int device, void* ptr) {
  DeviceScope scope(device);
  B200_CUDA(cudaIpcCloseMemHandle(ptr));
  return 0;
}
DEVA_B200_API int deva_b200_peer_free(int device, void* ptr) {
  DeviceScope scope(device);
  B200_CUDA(cudaFree(ptr));
  return 0;
}

}  // extern "C"
