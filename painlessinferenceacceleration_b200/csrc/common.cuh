// Shared host/device helpers of libpia_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <utility>

#include "../../include/pia_b200.h"

namespace pia {

void set_error(const char *fmt, ...);
extern std::atomic<unsigned long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

#define PIA_CUDA_CHECK(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      pia::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PIA_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

#define PIA_REQUIRE(cond, ...)          \
  do {                                  \
    if (!(cond)) {                      \
      pia::set_error(__VA_ARGS__);      \
      return PIA_ERR_INVALID;           \
    }                                   \
  } while (0)

// checks the launch itself (legal during stream capture: no sync)
#define PIA_LAUNCH_CHECK()                                                                  \
  do {                                                                                      \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      pia::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PIA_ERR_CUDA;                                                                  \
    }                                                                                       \
    pia::count_launch();                                                                    \
  } while (0)

constexpr unsigned FULL = 0xffffffffu;

// Programmatic dependent launch (PDL): every kernel of the decode step is launched with the
// programmatic-stream-serialization attribute, announces its dependents at once and waits for its predecessor
// (griddepcontrol.wait = predecessor complete + memory visible) before its first global access.  The next kernel's
// CTAs are then resident, with barriers set up, when the predecessor's last CTA retires, which hides the
// launch + prologue latency between the ~330 small kernels of a step.  PIA_PDL=0 disables the attribute (the
// device-side instructions are no-ops for a normally launched kernel).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

bool pdl_enabled();
extern thread_local int g_pdl_off;  // > 0: launches from this thread omit the PDL attribute (pia_gemm_plan_set_pdl)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                         cudaStream_t stream, unsigned cluster_x, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cluster_x > 1) {  // thread-block cluster along x (distributed shared memory between the CTAs of a cluster)
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster_x; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled() && g_pdl_off == 0) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args &&...args) {
  return launch_kernel_cluster(kernel, grid, block, smem, stream, 1u, std::forward<Args>(args)...);
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

}  // namespace pia
