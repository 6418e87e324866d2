// Shared host-side helpers of the C entry points: error slot, launch checks, casts from the ABI's types.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdio.h>

#include "deva_b200.h"

namespace b200 {

void set_error(const char* fmt, ...);  // stores into the thread-local slot read by deva_b200_last_error()

#define B200_REQUIRE(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      ::b200::set_error(__VA_ARGS__);    \
      return 1;                          \
    }                                    \
  } while (0)

#define B200_CUDA(expr)                                                              \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 2;                                                                      \
    }                                                                                \
  } while (0)

void count_launch();  // bumps the counter read by deva_b200_launch_count()
#define B200_LAUNCH_CHECK()          \
  do {                               \
    ::b200::count_launch();          \
    B200_CUDA(cudaGetLastError());   \
  } while (0)

inline int ceil_div(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// The ABI passes streams as deva_stream_t and fp16 buffers as void*.
inline cudaStream_t S(deva_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline __half* H(void* p) { return reinterpret_cast<__half*>(p); }
inline const __half* H(const void* p) { return reinterpret_cast<const __half*>(p); }

constexpr int kListCap = DEVA_B200_LIST_PITCH;  // max top_k; also the row pitch of the top-k index / weight lists

constexpr int kMaxDevices = 64;
int device_slot();  // current CUDA device, clamped to [0, kMaxDevices): index of per-device one-time state
int sm_count();  // cached multiprocessor count of the current device

}  // namespace b200
