// resblock_z.cu -- WNB_MATH_TF32 training forward of one residual block in "deferred skip" form.
//
// The reference block (wavenet.py:525-536) returns (x + res_1x1(z), skip_1x1(z)) and WaveNet.forward sums the
// skip outputs of all L blocks (wavenet.py:229-236).  Written per block, that sum costs a read-modify-write of the
// (B,T,S) skip accumulator in EVERY block -- 84 % of this block's HBM traffic at 64 res / 512 skip channels.
// The sum over blocks of z_l W2skip_l^T is one GEMM over the concatenated channel axis,
//      skip = [z_0 | z_1 | ... | z_{L-1}] [W2skip_0 | ... | W2skip_{L-1}]^T + sum_l b2skip_l ,
// so this kernel only writes z_l (into its 64-channel slice of Z_all (B,T,L*R)) and the residual output; the skip
// GEMM runs once after the last block (gemm_nt_tc, K = L*R).  Per block the traffic drops from 814 MB to 177 MB at
// the bench shape; Z_all (1.4 GB there) is also what the backward needs for the skip-weight gradient.
//
// Per 64-sample time tile (one consumer warpgroup, accumulators in registers):
//   GEMM-1  D1[64 x 128] = [x(t-d) | x(t) | aux(t)] [64 x 160] * W1^T      wgmma m64n128k8 tf32, both operands from
//                                                                          shared memory, W1 resident
//   gate    z = sigmoid(D1[:, :64] + b) * tanh(D1[:, 64:] + b)              registers -> swizzled staging tile -> Z_all
//   GEMM-2  D2[64 x 64]   = z * W2res^T                                     wgmma m64n64k8, A = the z staging tile
//   out     xout = D2 + b2res + x(t)   (x(t) is copied from the A stage into registers right after GEMM-1, so the A
//           stage is refilled while the gate / GEMM-2 / epilogue of this tile run)
// Roles (288 threads): two consumer warpgroups, each with its own A stage and staging tiles, working on alternate
// tiles (one's GEMMs overlap the other's epilogue); warp 8 = TMA producer (weights once, then the activation tiles
// of both warpgroups from a dynamic tile scheduler).  fp32 storage, tf32 multiplies, fp32 accumulate.
//
// Shared memory: W1 80 KB | W2res 16 KB | per warpgroup: A stage 40 KB, staging 16 KB.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace wnb {
namespace tcz {

constexpr int kTM = 64;
constexpr int kR = 64;
constexpr int kAp = 32;
constexpr int kK1 = 2 * kR + kAp;        // 160
constexpr int kSubBytes = kTM * 32 * 4;  // one [64 x 32 fp32] swizzled sub-tile
constexpr int kNSubA = kK1 / 32;         // 5
constexpr int kW1SubBytes = 2 * kR * 32 * 4;   // [128 x 32]
constexpr int kW2SubBytes = kR * 32 * 4;       // [64 x 32]
constexpr int kNWG = 2;
constexpr int kOffW1 = 0;
constexpr int kOffW2 = kOffW1 + kNSubA * kW1SubBytes;
constexpr int kOffA = kOffW2 + 2 * kW2SubBytes;
constexpr int kOffStg = kOffA + kNWG * kNSubA * kSubBytes;
constexpr int kOffBar = kOffStg + kNWG * 2 * kSubBytes;
constexpr int kSmemBytes = kOffBar + 256 + 1024;
constexpr int kThreadsZ = 128 * kNWG + 32;

struct alignas(64) Maps {
  CUtensorMap x, haux, w1, w2, xout, z;
};

enum { B_W = 0, B_AFULL0, B_AEMPTY0 = B_AFULL0 + kNWG, B_COUNT = B_AEMPTY0 + kNWG };

// dynamic tile scheduler: `sched` = {next tile, CTAs done}, two device words owned by the launching (device, stream)
// (common.cuh sched_counters): launches on different streams never share them.

__global__ void __launch_bounds__(kThreadsZ, 1)
resblock_fwd_z_kernel(const __grid_constant__ Maps maps, const float* __restrict__ b1, const float* __restrict__ b2,
                      int B, int T, int d, int has_xout, int zcol0, unsigned int* __restrict__ sched, int rev) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  volatile int* tile_slot = reinterpret_cast<volatile int*>(smem + kOffBar + 8 * B_COUNT);  // one per warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_b = (T + kTM - 1) / kTM;
  const int ntiles = B * tiles_per_b;

  if (threadIdx.x == 0) {
    ptx::mbar_init(&bars[B_W], 1);
    for (int g = 0; g < kNWG; g++) {
      ptx::mbar_init(&bars[B_AFULL0 + g], 1);
      ptx::mbar_init(&bars[B_AEMPTY0 + g], 128);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch: the set-up above overlapped the previous kernel's tail; from here on this
  // kernel reads / writes memory that kernel may have produced
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp == 4 * kNWG) {
    // =============================== TMA producer ===============================
    if (ptx::elect_one()) {
      ptx::prefetch_tmap(&maps.x); ptx::prefetch_tmap(&maps.haux);
      ptx::prefetch_tmap(&maps.w1); ptx::prefetch_tmap(&maps.w2);
      ptx::mbar_arrive_expect_tx(&bars[B_W], kNSubA * kW1SubBytes + (has_xout ? 2 * kW2SubBytes : 0));
      for (int j = 0; j < kNSubA; j++) ptx::tma_load_2d(smem + kOffW1 + j * kW1SubBytes, &maps.w1, &bars[B_W], j * 32, 0);
      if (has_xout) {
        ptx::tma_load_2d(smem + kOffW2, &maps.w2, &bars[B_W], 0, 0);
        ptx::tma_load_2d(smem + kOffW2 + kW2SubBytes, &maps.w2, &bars[B_W], 32, 0);
      }
      // rev: time tiles from the end of the tensor backwards -- a block whose producer ran front to back finds the rows
      // that block wrote LAST still in L2 (stack.cu alternates the direction from block to block)
      int tile = rev ? ntiles - 1 - (int)blockIdx.x : (int)blockIdx.x;
      if ((int)blockIdx.x >= ntiles) tile = -1;
      int stops = 0;
      for (uint32_t it = 0; stops < kNWG; it++) {
        const int g = it % kNWG;
        const uint32_t use = it / kNWG;
        ptx::mbar_wait(&bars[B_AEMPTY0 + g], (use & 1) ^ 1);
        tile_slot[g] = tile;                  // publish the tile (or the stop mark) to warpgroup g
        if (tile < 0) {
          ptx::mbar_arrive(&bars[B_AFULL0 + g]);
          stops++;
          continue;
        }
        const int b = tile / tiles_per_b, t0 = (tile - b * tiles_per_b) * kTM;
        ptx::mbar_arrive_expect_tx(&bars[B_AFULL0 + g], kNSubA * kSubBytes);
        unsigned char* sA = smem + kOffA + g * kNSubA * kSubBytes;
        ptx::tma_load_3d(sA + 0 * kSubBytes, &maps.x, &bars[B_AFULL0 + g], 0, t0 - d, b);
        ptx::tma_load_3d(sA + 1 * kSubBytes, &maps.x, &bars[B_AFULL0 + g], 32, t0 - d, b);
        ptx::tma_load_3d(sA + 2 * kSubBytes, &maps.x, &bars[B_AFULL0 + g], 0, t0, b);
        ptx::tma_load_3d(sA + 3 * kSubBytes, &maps.x, &bars[B_AFULL0 + g], 32, t0, b);
        ptx::tma_load_3d(sA + 4 * kSubBytes, &maps.haux, &bars[B_AFULL0 + g], 0, t0, b);
        tile = (int)(atomicAdd(&sched[0], 1u) + gridDim.x);
        if (tile >= ntiles) tile = -1;
        else if (rev) tile = ntiles - 1 - tile;
      }
    }
  } else {
    // =============================== consumer warpgroup g ===============================
    const int g = warp >> 2, wq = warp & 3, tid = threadIdx.x & 127;
    const int r0 = 16 * wq + (lane >> 2), cq = 2 * (lane & 3);   // fragment rows r0, r0 + 8; columns 8 j + cq (+1)
    unsigned char* sA = smem + kOffA + g * kNSubA * kSubBytes;
    unsigned char* stg = smem + kOffStg + g * 2 * kSubBytes;       // [64 x 64]: z, then xout, as two swizzled sub-tiles
    const uint32_t a_u32 = ptx::smem_u32(sA), w1_u32 = ptx::smem_u32(smem + kOffW1);
    const uint32_t w2_u32 = ptx::smem_u32(smem + kOffW2), stg_u32 = ptx::smem_u32(stg);
    const int bar_id = 1 + g;
    ptx::mbar_wait(&bars[B_W], 0);
    for (uint32_t j = 0;; j++) {
      ptx::mbar_wait(&bars[B_AFULL0 + g], j & 1);
      const int tile = tile_slot[g];
      if (tile < 0) break;
      const int b = tile / tiles_per_b, t0 = (tile - b * tiles_per_b) * kTM;
      // ---- GEMM-1 ----
      float d1[64];
#pragma unroll
      for (int i = 0; i < 64; i++) d1[i] = 0.f;
      ptx::wg_fence();
#pragma unroll
      for (int s = 0; s < kNSubA; s++)
#pragma unroll
        for (int k = 0; k < 4; k++)
          ptx::wgmma_ss<128>(d1, ptx::gmma_desc_k_sw128(a_u32 + s * kSubBytes + 32 * k),
                             ptx::gmma_desc_k_sw128(w1_u32 + s * kW1SubBytes + 32 * k), 1);
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_touch(d1);
      // ---- x(t) for the residual: A stage -> registers (fragment positions), then the stage can be refilled ----
      float xr[32];
      if (has_xout) {
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + cq;
          const float2 v = *reinterpret_cast<const float2*>(sA + (2 + (c >> 5)) * kSubBytes + ptx::sw128_off(r, c & 31));
          xr[i] = v.x; xr[i + 1] = v.y;
        }
      }
      ptx::mbar_arrive(&bars[B_AEMPTY0 + g]);
      // ---- gate: z = sigmoid(a) * tanh(g) on the fragments (column c and 64 + c are registers i and i + 32) ----
      float z[32];
#pragma unroll
      for (int i = 0; i < 32; i++) {
        const int c = 8 * (i >> 2) + cq + (i & 1);
        const float av = d1[i] + __ldg(b1 + c), tv = d1[i + 32] + __ldg(b1 + kR + c);
        z[i] = (0.5f * ptx::tanh_approx(0.5f * av) + 0.5f) * ptx::tanh_approx(tv);
      }
      // ---- z -> staging (the previous tile's xout store must have read it) -> Z_all slice ----
      if (tid == 0) ptx::bulk_wait_read<0>();
      ptx::named_bar(bar_id, 128);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + cq;
        *reinterpret_cast<float2*>(stg + (c >> 5) * kSubBytes + ptx::sw128_off(r, c & 31)) = make_float2(z[i], z[i + 1]);
      }
      ptx::fence_proxy_async();
      ptx::named_bar(bar_id, 128);
      if (tid == 0) {
        ptx::tma_store_3d(&maps.z, stg, zcol0, t0, b);
        ptx::tma_store_3d(&maps.z, stg + kSubBytes, zcol0 + 32, t0, b);
        ptx::bulk_commit();
      }
      if (!has_xout) continue;
      // ---- GEMM-2 from the z staging tile ----
      float d2[32];
#pragma unroll
      for (int i = 0; i < 32; i++) d2[i] = 0.f;
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 2; kk++)
#pragma unroll
        for (int k = 0; k < 4; k++)
          ptx::wgmma_ss<64>(d2, ptx::gmma_desc_k_sw128(stg_u32 + kk * kSubBytes + 32 * k),
                            ptx::gmma_desc_k_sw128(w2_u32 + kk * kW2SubBytes + 32 * k), 1);
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_touch(d2);
      // ---- residual output: xout = D2 + b2 + x(t), through the same staging tile once the z store has read it ----
      if (tid == 0) ptx::bulk_wait_read<0>();
      ptx::named_bar(bar_id, 128);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + cq;
        const float2 bv = __ldg(reinterpret_cast<const float2*>(b2 + c));
        *reinterpret_cast<float2*>(stg + (c >> 5) * kSubBytes + ptx::sw128_off(r, c & 31)) =
            make_float2(d2[i] + bv.x + xr[i], d2[i + 1] + bv.y + xr[i + 1]);
      }
      ptx::fence_proxy_async();
      ptx::named_bar(bar_id, 128);
      if (tid == 0) {
        ptx::tma_store_3d(&maps.xout, stg, 0, t0, b);
        ptx::tma_store_3d(&maps.xout, stg + kSubBytes, 32, t0, b);
        ptx::bulk_commit();
      }
    }
    if (tid == 0) ptx::bulk_wait<0>();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&sched[1], 1u) == gridDim.x - 1) {  // last CTA out: re-arm the scheduler for the next launch
      sched[0] = 0;
      sched[1] = 0;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Per-block form WITH skip accumulation (wnb_resblock_fwd, reference wavenet.py:525-536 one block at a time):
// GEMM-1 + gate as above, then the W2 row chunks -- [64 x 64] each: the residual chunk (unless this is the last
// block) and the S/64 skip chunks -- stream from L2 through a TMA ring and each is one wgmma m64n64 from the z staging
// tile: xout = D + b2 + x(t) (TMA store), skip += D + b2 (TMA reduce-add; TMA store when skip_init).  Every skip
// element receives exactly one add per launch.  One consumer warpgroup + one producer warp (W2 does not fit resident
// next to W1).  Shared memory: W1 80 KB | A stage 40 KB | z staging 16 KB | 2 output staging 32 KB | W2 ring 32 KB.
namespace tcs {
constexpr int kSNSlot = 2;
constexpr int kSChunkBytes = 2 * kW2SubBytes;                 // [64 rows x 64] as two [64 x 32] sub-tiles
constexpr int kSOffW1 = 0;
constexpr int kSOffA = kSOffW1 + kNSubA * kW1SubBytes;
constexpr int kSOffZ = kSOffA + kNSubA * kSubBytes;
constexpr int kSOffOut = kSOffZ + 2 * kSubBytes;
constexpr int kSOffRing = kSOffOut + 2 * 2 * kSubBytes;
constexpr int kSOffBar = kSOffRing + kSNSlot * kSChunkBytes;
constexpr int kSSmemBytes = kSOffBar + 256 + 1024;
constexpr int kSThreads = 128 + 32;
struct alignas(64) Maps { CUtensorMap x, haux, w1, w2, xout, skip; };
enum { SB_W = 0, SB_AFULL, SB_AEMPTY, SB_WF0, SB_WE0 = SB_WF0 + kSNSlot, SB_COUNT = SB_WE0 + kSNSlot };
}  // namespace tcs

__global__ void __launch_bounds__(tcs::kSThreads, 1)
resblock_fwd_skip_kernel(const __grid_constant__ tcs::Maps maps, const float* __restrict__ b1, const float* __restrict__ b2,
                         int B, int T, int S, int d, int has_xout, int skip_init, unsigned int* __restrict__ sched) {
  using namespace tcs;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kSOffBar);
  volatile int* tile_slot = reinterpret_cast<volatile int*>(smem + kSOffBar + 8 * SB_COUNT);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_b = (T + kTM - 1) / kTM;
  const int ntiles = B * tiles_per_b;
  const int nchunks = (has_xout ? 1 : 0) + S / 64;
  const int row0 = has_xout ? 0 : kR;      // first W2 row of chunk 0

  if (threadIdx.x == 0) {
    ptx::mbar_init(&bars[SB_W], 1);
    ptx::mbar_init(&bars[SB_AFULL], 1);
    ptx::mbar_init(&bars[SB_AEMPTY], 128);
    for (int i = 0; i < kSNSlot; i++) { ptx::mbar_init(&bars[SB_WF0 + i], 1); ptx::mbar_init(&bars[SB_WE0 + i], 128); }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp == 4) {
    // =============================== TMA producer: W1 once, then per tile the A stage and the W2 chunks ===============
    if (ptx::elect_one()) {
      ptx::prefetch_tmap(&maps.x); ptx::prefetch_tmap(&maps.haux); ptx::prefetch_tmap(&maps.w1); ptx::prefetch_tmap(&maps.w2);
      ptx::mbar_arrive_expect_tx(&bars[SB_W], kNSubA * kW1SubBytes);
      for (int j = 0; j < kNSubA; j++) ptx::tma_load_2d(smem + kSOffW1 + j * kW1SubBytes, &maps.w1, &bars[SB_W], j * 32, 0);
      int tile = (int)blockIdx.x < ntiles ? (int)blockIdx.x : -1;
      uint32_t slot = 0, wph = 0;
      for (uint32_t it = 0;; it++) {
        ptx::mbar_wait(&bars[SB_AEMPTY], (it & 1) ^ 1);
        tile_slot[0] = tile;
        if (tile < 0) { ptx::mbar_arrive(&bars[SB_AFULL]); break; }
        const int b = tile / tiles_per_b, t0 = (tile - b * tiles_per_b) * kTM;
        ptx::mbar_arrive_expect_tx(&bars[SB_AFULL], kNSubA * kSubBytes);
        unsigned char* sA = smem + kSOffA;
        ptx::tma_load_3d(sA + 0 * kSubBytes, &maps.x, &bars[SB_AFULL], 0, t0 - d, b);
        ptx::tma_load_3d(sA + 1 * kSubBytes, &maps.x, &bars[SB_AFULL], 32, t0 - d, b);
        ptx::tma_load_3d(sA + 2 * kSubBytes, &maps.x, &bars[SB_AFULL], 0, t0, b);
        ptx::tma_load_3d(sA + 3 * kSubBytes, &maps.x, &bars[SB_AFULL], 32, t0, b);
        ptx::tma_load_3d(sA + 4 * kSubBytes, &maps.haux, &bars[SB_AFULL], 0, t0, b);
        for (int c = 0; c < nchunks; c++) {
          ptx::mbar_wait(&bars[SB_WE0 + slot], wph ^ 1);
          ptx::mbar_arrive_expect_tx(&bars[SB_WF0 + slot], kSChunkBytes);
          unsigned char* dst = smem + kSOffRing + slot * kSChunkBytes;
          ptx::tma_load_2d(dst, &maps.w2, &bars[SB_WF0 + slot], 0, row0 + c * 64);
          ptx::tma_load_2d(dst + kW2SubBytes, &maps.w2, &bars[SB_WF0 + slot], 32, row0 + c * 64);
          if (++slot == kSNSlot) { slot = 0; wph ^= 1; }
        }
        tile = (int)(atomicAdd(&sched[0], 1u) + gridDim.x);
        if (tile >= ntiles) tile = -1;
      }
    }
  } else {
    // =============================== consumer warpgroup ===============================
    const int wq = warp & 3, tid = threadIdx.x;
    const int r0 = 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
    unsigned char* sA = smem + kSOffA;
    unsigned char* zst = smem + kSOffZ;
    const uint32_t a_u32 = ptx::smem_u32(sA), w1_u32 = ptx::smem_u32(smem + kSOffW1), z_u32 = ptx::smem_u32(zst);
    uint32_t slot = 0, wph = 0, nout = 0;
    ptx::mbar_wait(&bars[SB_W], 0);
    for (uint32_t j = 0;; j++) {
      ptx::mbar_wait(&bars[SB_AFULL], j & 1);
      const int tile = tile_slot[0];
      if (tile < 0) break;
      const int b = tile / tiles_per_b, t0 = (tile - b * tiles_per_b) * kTM;
      float d1[64];
#pragma unroll
      for (int i = 0; i < 64; i++) d1[i] = 0.f;
      ptx::wg_fence();
#pragma unroll
      for (int s = 0; s < kNSubA; s++)
#pragma unroll
        for (int k = 0; k < 4; k++)
          ptx::wgmma_ss<128>(d1, ptx::gmma_desc_k_sw128(a_u32 + s * kSubBytes + 32 * k),
                             ptx::gmma_desc_k_sw128(w1_u32 + s * kW1SubBytes + 32 * k), 1);
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_touch(d1);
      float xr[32];
      if (has_xout) {
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + cq;
          const float2 v = *reinterpret_cast<const float2*>(sA + (2 + (c >> 5)) * kSubBytes + ptx::sw128_off(r, c & 31));
          xr[i] = v.x; xr[i + 1] = v.y;
        }
      }
      ptx::mbar_arrive(&bars[SB_AEMPTY]);
      // ---- gate -> z staging tile (the A operand of every W2 chunk; the previous tile's MMAs have all completed) ----
      ptx::named_bar(1, 128);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + cq;
        float zz[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const float av = d1[i + h] + __ldg(b1 + c + h), tv = d1[i + h + 32] + __ldg(b1 + kR + c + h);
          zz[h] = (0.5f * ptx::tanh_approx(0.5f * av) + 0.5f) * ptx::tanh_approx(tv);
        }
        *reinterpret_cast<float2*>(zst + (c >> 5) * kSubBytes + ptx::sw128_off(r, c & 31)) = make_float2(zz[0], zz[1]);
      }
      ptx::fence_proxy_async();
      ptx::named_bar(1, 128);
      // ---- W2 chunks: residual (unless last block), then skip ----
      for (int c = 0; c < nchunks; c++) {
        const bool is_res = has_xout && c == 0;
        const int col0 = is_res ? 0 : (c - (has_xout ? 1 : 0)) * 64;   // channel offset inside xout / skip
        const float* bias = b2 + (is_res ? 0 : kR + col0);
        ptx::mbar_wait(&bars[SB_WF0 + slot], wph);
        const uint32_t w_u32 = ptx::smem_u32(smem + kSOffRing + slot * kSChunkBytes);
        float d2[32];
#pragma unroll
        for (int i = 0; i < 32; i++) d2[i] = 0.f;
        ptx::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 2; kk++)
#pragma unroll
          for (int k = 0; k < 4; k++)
            ptx::wgmma_ss<64>(d2, ptx::gmma_desc_k_sw128(z_u32 + kk * kSubBytes + 32 * k),
                              ptx::gmma_desc_k_sw128(w_u32 + kk * kW2SubBytes + 32 * k), 1);
        ptx::wg_commit();
        ptx::wg_wait<0>();
        ptx::wg_touch(d2);
        ptx::mbar_arrive(&bars[SB_WE0 + slot]);
        if (++slot == kSNSlot) { slot = 0; wph ^= 1; }
        unsigned char* ost = smem + kSOffOut + (nout & 1) * 2 * kSubBytes;
        if (tid == 0) ptx::bulk_wait_read<1>();   // the store that last read this staging tile has drained
        ptx::named_bar(1, 128);
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int r = r0 + 8 * ((i >> 1) & 1), cc = 8 * (i >> 2) + cq;
          const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + cc));
          float v0 = d2[i] + bv.x, v1 = d2[i + 1] + bv.y;
          if (is_res) { v0 += xr[i]; v1 += xr[i + 1]; }
          *reinterpret_cast<float2*>(ost + (cc >> 5) * kSubBytes + ptx::sw128_off(r, cc & 31)) = make_float2(v0, v1);
        }
        ptx::fence_proxy_async();
        ptx::named_bar(1, 128);
        if (tid == 0) {
          for (int h = 0; h < 2; h++) {
            if (is_res) ptx::tma_store_3d(&maps.xout, ost + h * kSubBytes, 32 * h, t0, b);
            else if (skip_init) ptx::tma_store_3d(&maps.skip, ost + h * kSubBytes, col0 + 32 * h, t0, b);
            else ptx::tma_reduce_add_3d(&maps.skip, ost + h * kSubBytes, col0 + 32 * h, t0, b);
          }
          ptx::bulk_commit();
        }
        nout++;
      }
    }
    if (tid == 0) ptx::bulk_wait<0>();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&sched[1], 1u) == gridDim.x - 1) {  // last CTA out: re-arm the scheduler for the next launch
      sched[0] = 0;
      sched[1] = 0;
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// fp32 (B, T, C) view with row pitch ld floats (ld >= C: a channel slice of a wider tensor), box [32 x rows x 1]
static bool map_act(CUtensorMap* m, const void* base, int C, int ld, int T, int B, int rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B};
  cuuint64_t gstr[2] = {(cuuint64_t)ld * 4, (cuuint64_t)ld * 4 * (cuuint64_t)T};
  cuuint32_t box[3] = {32, (cuuint32_t)rows, 1}, es[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// fp32 row-major matrix (rows x cols), box [32 x box_rows]
static bool map_mat(CUtensorMap* m, const void* base, int cols, int rows, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows}, es[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tcz

bool resblock_fwd_z_supported(int R, int Ap, int ks) { return R == tcz::kR && ks == 2 && Ap == tcz::kAp; }

// One block in deferred-skip form: xout (B,T,R) or null (last block), z -> zall[:, :, zcol0 : zcol0+R] (row pitch ldz).
int resblock_fwd_z(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2res,
                   const float* b2res, float* xout, float* zall, int ldz, int zcol0, int B, int T, int d,
                   cudaStream_t st, int reverse) {
  using namespace tcz;
  if ((reinterpret_cast<uintptr_t>(b1) | reinterpret_cast<uintptr_t>(b2res)) & 15) {
    set_error("resblock_fwd_z: b1 / b2 must be 16-byte aligned");
    return WNB_ERR_INVALID;
  }
  Maps maps;
  bool ok = map_act(&maps.x, xin, kR, kR, T, B, kTM) && map_act(&maps.haux, haux, kAp, kAp, T, B, kTM) &&
            map_mat(&maps.w1, w1, kK1, 2 * kR, 2 * kR) && map_mat(&maps.w2, w2res ? w2res : w1, kR, kR, kR) &&
            map_act(&maps.xout, xout ? xout : xin, kR, kR, T, B, kTM) && map_act(&maps.z, zall, ldz, ldz, T, B, kTM);
  if (!ok) {
    set_error("resblock_fwd_z: cuTensorMapEncodeTiled failed or is unavailable");
    return WNB_ERR_CUDA;
  }
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(resblock_fwd_z_kernel), kSmemBytes));
  const int sms = device_sms();
  unsigned int* sched = sched_counters(st);
  if (!sched) { set_error("resblock_fwd_z: cannot allocate the scheduler words"); return WNB_ERR_CUDA; }
  const int ntiles = B * ((T + kTM - 1) / kTM);
  const int grid = ntiles < sms ? ntiles : sms;
  if (launch_pdl(resblock_fwd_z_kernel, grid, kThreadsZ, kSmemBytes, st, 1, maps, b1, b2res ? b2res : b1, B, T, d,
                 xout ? 1 : 0, zcol0, sched, reverse ? 1 : 0) != cudaSuccess) { /* reported below */ }
  WNB_CHECK_LAUNCH("resblock_fwd_z");
  return WNB_OK;
}

bool resblock_fwd_skip_supported(int R, int S, int Ap, int ks) {
  return R == tcz::kR && ks == 2 && Ap == tcz::kAp && S >= 64 && S % 64 == 0;
}

// One block in the per-block form: xout (B,T,R) or null (last block), skip (B,T,S) = or += the block's skip output.
int resblock_fwd_skip(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2,
                      const float* b2, float* xout, float* skip, int B, int T, int S, int d, int skip_init,
                      cudaStream_t st) {
  using namespace tcz;
  if ((reinterpret_cast<uintptr_t>(b1) | reinterpret_cast<uintptr_t>(b2)) & 15) {
    set_error("resblock_fwd: b1 / b2 must be 16-byte aligned");
    return WNB_ERR_INVALID;
  }
  tcs::Maps maps;
  bool ok = map_act(&maps.x, xin, kR, kR, T, B, kTM) && map_act(&maps.haux, haux, kAp, kAp, T, B, kTM) &&
            map_mat(&maps.w1, w1, kK1, 2 * kR, 2 * kR) && map_mat(&maps.w2, w2, kR, kR + S, kR) &&
            map_act(&maps.xout, xout ? xout : xin, kR, kR, T, B, kTM) && map_act(&maps.skip, skip, S, S, T, B, kTM);
  if (!ok) {
    set_error("resblock_fwd: cuTensorMapEncodeTiled failed or is unavailable");
    return WNB_ERR_CUDA;
  }
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(resblock_fwd_skip_kernel), tcs::kSSmemBytes));
  const int sms = device_sms();
  unsigned int* sched = sched_counters(st);
  if (!sched) { set_error("resblock_fwd: cannot allocate the scheduler words"); return WNB_ERR_CUDA; }
  const int ntiles = B * ((T + kTM - 1) / kTM);
  const int grid = ntiles < sms ? ntiles : sms;
  if (launch_pdl(resblock_fwd_skip_kernel, grid, tcs::kSThreads, tcs::kSSmemBytes, st, 1, maps, b1, b2, B, T, S, d,
                 xout ? 1 : 0, skip_init, sched) != cudaSuccess) { /* reported below */ }
  WNB_CHECK_LAUNCH("resblock_fwd_skip");
  return WNB_OK;
}

}  // namespace wnb
