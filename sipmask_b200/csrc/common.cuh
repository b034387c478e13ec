// Shared helpers for the sipmask_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <stdlib.h>

#include "../../include/sipmask_b200.h"

namespace smb {

void set_error(const char* fmt, ...);

#define SMB_CHECK_ARG(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      smb::set_error(__VA_ARGS__);               \
      return SMB_EINVAL;                         \
    }                                            \
  } while (0)

#define SMB_CUDA_OK(expr)                                                            \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      smb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SMB_ECUDA;                                                              \
    }                                                                                \
  } while (0)

#define SMB_LAUNCH_OK(name)                                                          \
  do {                                                                               \
    cudaError_t _e = cudaGetLastError();                                             \
    if (_e != cudaSuccess) {                                                         \
      smb::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));       \
      return SMB_ECUDA;                                                              \
    }                                                                                \
  } while (0)

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is PER DEVICE: a process that drives several GPUs must opt in on
// each of them.  `static DeviceOnce once; if (once.first()) { ...set attributes... }` runs the body once per device.
struct DeviceOnce {
  bool done[64];
  DeviceOnce() { memset(done, 0, sizeof(done)); }
  bool first() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;   // unknown device: always (cheap) set
    if (done[dev]) return false;
    done[dev] = true;
    return true;
  }
};

// Programmatic dependent launch (PDL).  The elementwise / NMS kernels are launched with plain <<<>>>, so for them
// griddepcontrol.wait is a no-op (the stream already orders them after the previous kernel).  launch_dependents is not:
// smb_conv_run launches conv_gemm_kernel with the PDL attribute, and the signal lets that next convolution be scheduled
// and run its prologue (shared-memory carve-up, mbarrier init) while this kernel is still running.  The convolution
// executes griddepcontrol.wait before it touches global memory, so it still sees every write of this kernel.
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// GroupNorm statistics are accumulated as 64-bit fixed point (deterministic integer atomics)
constexpr float kGnSumScale = 1048576.0f;   // 2^20
constexpr float kGnSqScale = 65536.0f;      // 2^16

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

}  // namespace smb
