// tc_ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) async machinery of the tensor-core kernels:
// mbarrier, TMA (cp.async.bulk.tensor load / store / reduce-add), wgmma (fences, commit / wait groups, shared-memory
// matrix descriptors; the MMA wrappers themselves are in wgmma_tf32.cuh and wgmma_bf16.cuh), named barriers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma_bf16.cuh"
#include "wgmma_tf32.cuh"

namespace wnb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- programmatic dependent launch
// Kernels launched with launch_pdl() (common.cuh) may become resident while the previous kernel of the stream is
// still draining: everything up to pdl_wait() (barrier init, tensor-map prefetch) overlaps that
// kernel's tail; pdl_wait() returns once the previous kernel has completed and its writes are visible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same shared-memory offset as `bar` in CTA `rank` of the cluster.  Default (.release.cta)
// semantics: this releases a stage whose shared-memory reads are already complete (wgmma wait_group), so no cluster-scope
// release is needed -- .release.cluster would put a MEMBAR.ALL.GPU in front of every arrive.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// every thread of every CTA of the cluster; makes barrier initialisation and shared-memory writes visible cluster-wide
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded waits: a protocol bug must trap (error returned to the host) instead of hanging the GPU -- but the bound is
// WALL-CLOCK time (20 s on %globaltimer, looked at every 64 K polls), not a poll count: under a profiler's kernel
// replay, time slicing or preemption a healthy kernel can sit on a barrier for many millions of polls.
// The time-out path makes no function call unless WNB_WAIT_PRINTF is defined (a debugging build that prints the block
// and thread of the time-out): a call (printf) inside a wgmma pipeline makes ptxas serialise every wgmma.mma_async of
// the kernel (note C7510), which is what the tensor-core kernels would pay for the message in every build.
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
struct SpinGuard {
  uint32_t polls = 0;
  uint64_t t0 = 0;
  __device__ __forceinline__ bool expired() {
    if ((++polls & 0xFFFFu) != 0) return false;
    const uint64_t now = globaltimer_ns();
    if (t0 == 0) { t0 = now; return false; }
    return now - t0 > 20000000000ull;
  }
};
// A kernel that sets per-warpgroup register budgets (setmaxnreg) ends a timed-out wait with kStoreFault: a store to
// address 0, which the host sees as an illegal-address error.  A trap instruction anywhere in such a kernel makes ptxas
// allocate every warpgroup at the launch bound instead of its setmaxnreg budget.
enum WaitTimeout { kTrap = 0, kStoreFault = 1 };
template <int kOnTimeout = kTrap>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  SpinGuard guard;
  while (!mbar_try_wait(bar, parity)) {
    if (guard.expired()) {
#ifdef WNB_WAIT_PRINTF
      printf("wnb200: mbarrier wait timed out after 20 s (block %d thread %d)\n", blockIdx.x, threadIdx.x);
#endif
      if (kOnTimeout == kStoreFault) *reinterpret_cast<volatile int*>(0) = 0;
      else __trap();
    }
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// the same box written to the same shared-memory offset of every CTA of the cluster in `cta_mask`; each destination's
// barrier at `bar`'s offset receives the box's bytes
__device__ __forceinline__ void tma_load_2d_multicast(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// L2 prefetch of a box (no shared-memory destination, no barrier): shortens the latency of the load that follows
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* m, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];"
               ::"l"((uint64_t)m), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"((uint64_t)m), "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"((uint64_t)m), "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void st_shared_v4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor of a K-major operand tile in the 128B-swizzled layout TMA writes with
// CU_TENSOR_MAP_SWIZZLE_128B: rows of 32 fp32 (128 B), 8-row groups 1024 B apart (SBO), LBO unused.  The tile must start
// on a 1024-byte boundary; the k-th group of 8 tf32 inside the row is addressed by adding 32 k bytes (2 k in the
// descriptor's 16-byte units) to the start address.
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// The same for a K-major bf16 tile in the 64B-swizzled layout (CU_TENSOR_MAP_SWIZZLE_64B): rows of 32 bf16 (64 B),
// 8-row groups 512 B apart, tile start on a 512-byte boundary; the k-th group of 16 bf16 is at +32 k bytes.
__device__ __forceinline__ uint64_t gmma_desc_k_sw64(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (32ull << 32) | (2ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma wait
template <int R>
__device__ __forceinline__ void wg_touch(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// per-thread register budget of the executing warpgroup (every thread of it executes the same call): a producer
// warpgroup hands registers back so that the consumer warpgroups can take more than the launch bound gives
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// barrier over `threads` threads (a multiple of 32) of the CTA; id 0 is __syncthreads
__device__ __forceinline__ void named_bar(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// byte offset of element (row r, column c < 32) in a [rows x 32 fp32] tile written by TMA with 128B swizzle
__host__ __device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)(r * 128 + ((((c >> 2) ^ r) & 7) << 4) + ((c & 3) << 2));
}

// byte offset of element (row n, column k < 32) in a [rows x 32 bf16] tile in the 64B-swizzled layout
__device__ __forceinline__ uint32_t sw64_off(int n, int k) {
  return (uint32_t)(n * 64 + ((((k >> 3) ^ (n >> 1)) & 3) << 4) + ((k & 7) << 1));
}
// two fp32 -> one register of two bf16, each rounded to nearest even; lo goes to the lower half
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace ptx
}  // namespace wnb
