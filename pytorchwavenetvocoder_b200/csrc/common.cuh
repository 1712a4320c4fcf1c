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
enum { SCRATCH_WGRAD = 0, SCRATCH_EMBED = 1, SCRATCH_AUX = 2, SCRATCH_LOSS = 3, SCRATCH_EMBED_PART = 4, SCRATCH_BF16 = 5,
       SCRATCH_SIMT = 6 };

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

// The window of one resumable decode call (the four decode _at launchers, include/wnb200.h).  The kernels keep absolute
// indices: the launcher shifts xs by -xs_base columns, h by -h_frame0 columns, uniforms by -i0 columns and logits_out by
// -i0 rows, so that a kernel reads position pp at xs[.. + pp], frame f at h[.. + f], and sample i's uniform and logits at
// i; n_samples become absolute ends (i0 + n_b).  A one-shot call is the window pos0 = xs_base = h_frame0 = 0.
struct DecodeWindow {
  int pos0, i0;      // first position; first sample index = max(pos0 - (P - 1), 0)
  int i_last;        // i0 + max_n - 1: the last sample index the call may generate (the uniforms clamp)
  int h_last;        // h_frame0 + Th - 1: the last frame of h (lookups past it are clamped to it)
  int stride_xs;     // xs row stride: columns xs_base .. max(pos0, P - 1) + max_n
};
template <class T>
static inline T* shift_ptr(T* ptr, long long n) {   // ptr + n elements, NULL stays NULL (n may be negative)
  return ptr ? reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(ptr) + (uintptr_t)(n * (long long)sizeof(T))) : ptr;
}
// False (message set) when the window is inconsistent or its positions would not fit an int.
static inline bool decode_window(const char* name, int P, int n_pad, int U, int ks, int max_n, int Th, int pos0,
                                 int xs_base, int h_frame0, DecodeWindow* w) {
  const int first = pos0 - (ks - 1) > 0 ? pos0 - (ks - 1) : 0;            // oldest column the front gather reads
  const int j0 = pos0 - n_pad > 0 ? pos0 - n_pad : 0;                      // aux column of pos0
  const int f0 = U > 0 ? j0 / U : j0;                                      // its frame
  const long long last = (long long)(pos0 > P - 1 ? pos0 : P - 1) + max_n;  // last xs column written
  // a call generates at least one sample, so a chain of calls never starts one inside the warm-up: pos0 is 0 (the first
  // call) or past it
  if (pos0 < 0 || (pos0 > 0 && pos0 < P - 1) || xs_base < 0 || xs_base > first || h_frame0 < 0 || h_frame0 > f0 ||
      last >= 0x7fffffffLL || (long long)h_frame0 + Th > 0x7fffffffLL) {
    set_error("%s: bad window (pos0 %d, xs_base %d, h_frame0 %d, P %d, n_pad %d, max_n %d)", name, pos0, xs_base,
              h_frame0, P, n_pad, max_n);
    return false;
  }
  w->pos0 = pos0;
  w->i0 = pos0 > P - 1 ? pos0 - (P - 1) : 0;
  w->i_last = w->i0 + max_n - 1;
  w->h_last = h_frame0 + Th - 1;
  w->stride_xs = (int)(last + 1 - xs_base);
  return true;
}

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

// Inverse-CDF pick of the three decode kernels, called by all 32 lanes of a warp.  Each lane owns consecutive classes
// (lane order = class order) with e_q = expf(l_q - max) summing to `lsum`; `incl` is the inclusive shuffle scan of the
// lanes' lsum, `lnz` the lane's last class with e_q > 0 (-1 if none), `uni` in [0, 1).  `walk(start, target)` returns
// the lane's first class with e_q > 0 whose running sum from start passes target, or -1.
// A lane claims target = uni * total when excl <= target < incl, with excl = the previous lane's incl (0 on lane 0):
// bit-equal neighbours, so no target below the total falls between two lanes.  The scan's sums are not monotone in
// the lane (a lane of zero mass can end a rounding step above its predecessor), but the first lane whose incl exceeds
// the target always claims it, and overlapping claims take the lowest class.  The walk starts from incl - lsum, which
// can differ from excl by rounding: every target that lane's own interval [incl - lsum, incl) held before the claim
// test used excl picks what it picked then.  A walk that never passes the target picks the last class with e_q > 0 at
// or before its lane; a target no lane claims (>= total), the row's last such class.  So the pick always has nonzero
// probability.
template <class Walk>
__device__ __forceinline__ int sample_pick(float incl, float lsum, int lnz, float uni, int lane, Walk walk) {
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 0.f;
  const float total = __shfl_sync(0xffffffffu, incl, 31);
  const float target = uni * total;
  const bool claim = target >= excl && target < incl;
  int cand = claim ? walk(incl - lsum, target) : 0x7fffffff;
  const bool fell = cand < 0;
  const unsigned claims = __ballot_sync(0xffffffffu, claim);
  if (claims == 0u || __any_sync(0xffffffffu, fell)) {   // rare: a target within rounding of a lane's upper end
    int pl = lnz;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, pl, o);
      if (lane >= o) pl = max(pl, v);
    }
    if (fell) cand = pl;
    if (claims == 0u) cand = __shfl_sync(0xffffffffu, pl, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
  return cand;
}

}  // namespace wnb
