// common.cuh -- error plumbing and small device helpers shared by every kernel file of libwnb200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/wnb200.h"

namespace wnb {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// Optional per-launch CUDA-event timing by kernel kind (WNB_PROF_* in wnb200.h), see wnb_profile_enable().
void prof_begin(int kind, cudaStream_t st);
void prof_end(int kind, cudaStream_t st);
struct ProfScope {
  int kind; cudaStream_t st;
  ProfScope(int k, cudaStream_t s) : kind(k), st(s) { prof_begin(k, s); }
  ~ProfScope() { prof_end(kind, st); }
};

// Launch with programmatic stream serialization (PDL): the kernel may become resident while its predecessor in the
// stream drains; it must call ptx::pdl_wait() before touching global memory (all kernels launched this way do).
// WNB_PDL=0 in the environment turns the attribute off.  cluster > 1: thread-block clusters of `cluster` CTAs along x
// (grid a multiple of it).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t st,
                              unsigned cluster, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster > 1 ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- per-device / per-stream launch state (thread-safe; elementwise.cu) -------------------------------------------
// SM count of the CURRENT device (cached per device).
int device_sms();
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (device, kernel) -- function attributes are per device.
cudaError_t ensure_dynamic_smem(const void* func, size_t bytes);
// Two zero-initialised uint32 words of device memory owned by (current device, stream): the dynamic tile scheduler
// of the block kernels (tile counter, CTAs-done counter; the last CTA re-arms them).  Launches on DIFFERENT streams
// get different words and may run concurrently; launches on one stream are ordered.  A few bytes per stream, allocated
// on first use and kept for the life of the process (library state, not a caller-visible buffer).
unsigned int* sched_counters(cudaStream_t st);
// Device scratch owned by (current device, stream, slot), grown on demand (an outgrown buffer stays allocated, so a
// pointer handed out earlier remains valid).  Used for the per-CTA partial sums that make the gradient reductions independent of scheduling,
// and for the bf16 copies of the weights a WNB_MATH_BF16 call multiplies with.
void* scratch_buffer(cudaStream_t st, int slot, size_t bytes);
enum { SCRATCH_WGRAD = 0, SCRATCH_EMBED = 1, SCRATCH_AUX = 2, SCRATCH_LOSS = 3, SCRATCH_EMBED_PART = 4, SCRATCH_BF16 = 5 };

#define WNB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::wnb::set_error(__VA_ARGS__);      \
      return WNB_ERR_INVALID;             \
    }                                     \
  } while (0)

#define WNB_CHECK_LAUNCH(name)                                                     \
  do {                                                                             \
    cudaError_t e__ = cudaGetLastError();                                          \
    if (e__ != cudaSuccess) {                                                      \
      ::wnb::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));    \
      return WNB_ERR_CUDA;                                                         \
    }                                                                              \
    ::wnb::count_launch();                                                         \
  } while (0)

#define WNB_CUDA(call)                                                             \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) {                                                      \
      ::wnb::set_error("%s failed: %s", #call, cudaGetErrorString(e__));           \
      return WNB_ERR_CUDA;                                                         \
    }                                                                              \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace wnb
