// wgrad_tc.cu -- tensor-core weight gradients:  C[m][n] += sum_{b,t} A[b][t][m] * Bm[b][t+shift][n]
//
// The reduction index is TIME.  With channels-last activations a TMA box [32 time rows x 32 channels] is an MN-major
// tile, and Hopper's tf32 wgmma takes K-major operands only.  So per 32-step stage the two consumer warpgroups
//   - transpose the B sub-tiles (up to 7 x 32 channels) into one K-major [N x 32] tile in shared memory, and
//   - read their A fragments (64 of the 128 M-block rows each) straight from the swizzled A sub-tiles into registers,
// then issue wgmma m64nNk8 (A from registers, B from shared memory; double-buffered, so the transpose of the next stage
// overlaps the MMAs of this one) into an fp32 accumulator that stays in registers for ALL time tiles a CTA owns.  At the
// end every CTA writes its accumulator to its own slot of a scratch buffer and wgrad_reduce_kernel adds the slots of a
// segment into C in slot order: no atomics, so the gradients do not depend on how the CTAs were scheduled.
// A third role, one producer warp, streams the stages with TMA through an mbarrier ring.
// Launch shapes: up to 5 M-blocks sharing one B operand (one CTA set per M-block); column groups of B across CTAs
// (n_split, A shared through L2); segments = many independent problems of one structure (every residual block's dW1)
// in one launch, `ksplit` CTAs per segment, each on a contiguous range of its time tiles.
//
// Generic over "sub-tile lists": A = 4 groups of 32 channels (M = 128), B = up to 7 groups (N <= 224),
// each group = (tensor map, channel offset, time shift); dilated taps are just shifted groups, zero filled
// out of range by TMA.  An optional extra all-ones B group turns column 0 of that group into the bias
// gradient sum_t A[t][m] (replaces colsum_kernel).
//
// bf16 operands (BF16 = true, WgOpts::bf16): the transpose writes B rounded to bf16 (cvt.rn.bf16x2 of two time rows)
// into a 64B-swizzled K-major [N x 32] bf16 tile, the A fragments are rounded the same way from the fp32 sub-tiles, and
// the MMAs are bf16 wgmma m64nNk16 with fp32 accumulation.  The all-ones rows are exact in bf16; slots and their
// reduction are unchanged.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace wnb {
namespace wg {

constexpr int kMaxMB = 5;                    // M-blocks (128 rows each) sharing one B operand per launch
constexpr int kMaxB = 8, kMaxMaps = 6, kMaxOps = 2 * kMaxMB + 8;
constexpr int kConsumers = 256;              // two warpgroups: rows 0..63 and 64..127 of the M-block
constexpr int kThreadsW = kConsumers + 32;
constexpr int kMaxSeg = 64;
constexpr int kTK = 32;                      // time rows per stage (K of one stage)
constexpr int kSub = kTK * 128;              // one [32 x 32 fp32] swizzled sub-tile

// One TMA load per operand and stage: the tensor (B,T,C) is mapped 4-D as {32 ch, T, C/32 groups, B} with a box of
// {32, 32, groups, 1}, which lands in shared memory as `groups` consecutive [32 x 32] swizzled sub-tiles.
struct Op { int map; int cgrp0; int shift; int flags; int seg_cgrp_stride; int dst_group; };   // flags: WG_* of tc_host.h
struct alignas(64) Params {
  CUtensorMap maps[kMaxMaps];
  Op ops[kMaxOps]; int nops;     // A operands of every M-block (4 groups each), then the B operands
  int nMB, nB, use_ones;         // nB excludes the ones group
  float* c[kMaxMB]; int ldc;     // per block: C rows m (0..127), columns n (0..32*nB-1)
  int m_valid[kMaxMB];           // rows >= m_valid are padding (not written)
  float* db[kMaxMB];             // per block (128) or null
  int T, B, tiles_per_b, ntiles, nstages;
  int n_split;                   // column groups of the B operand handled by different CTAs (WgOpts)
  int ksplit;                    // CTAs per (M-block, column group, segment), each on a contiguous range of time tiles
  float* part;                   // one [128 x N] accumulator slot per CTA
  int ncols;                     // N: columns of a slot (32 * nB, + 32 for the ones group)
  int nseg, c_seg_stride, db_seg_stride;
  int seg_shift[kMaxSeg];
};

// bytes of one row (32 time steps) of the transposed B tile
template <bool BF16>
__host__ __device__ constexpr int bt_row_bytes() { return BF16 ? 64 : 128; }

template <int N, bool BF16>
__global__ void __launch_bounds__(kThreadsW, 1) wgrad_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int kBtRow = bt_row_bytes<BF16>();
  const int stage_bytes = (4 + p.nB) * kSub;
  unsigned char* bT = smem;                                   // 2 x K-major [N x 32] B tile (+ the ones rows)
  unsigned char* ring = smem + 2 * N * kBtRow;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)p.nstages * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.nstages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // CTA -> (M-block, column group, segment, time split); with n_split column groups neighbouring CTAs stream the same
  // time range (A operand shared through L2) for different 32*nB-channel groups of the B operand.  Tiles are indexed
  // f = seg * ntiles + tile; a CTA's range lies inside one segment.
  const int mb = blockIdx.x % p.nMB;
  const int rest = blockIdx.x / p.nMB;
  const int ng = rest % p.n_split, r2 = rest / p.n_split;
  const int seg0 = r2 / p.ksplit, tsplit = r2 % p.ksplit;
  const int bcol0 = ng * 32 * p.nB;
  const int per = (p.ntiles + p.ksplit - 1) / p.ksplit;
  const int tile_begin = seg0 * p.ntiles + min(p.ntiles, tsplit * per);
  const int tile_end = seg0 * p.ntiles + min(p.ntiles, (tsplit + 1) * per);

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kConsumers);
    }
    ptx::fence_barrier_init();
  }
  if (p.use_ones) {   // the ones rows of both transposed B tiles: filled once, never overwritten
    for (int h = 0; h < 2; h++) {
      if constexpr (BF16) {
        uint4* o = reinterpret_cast<uint4*>(bT + h * N * kBtRow + p.nB * 32 * kBtRow);
        for (int i = threadIdx.x; i < 32 * kBtRow / 16; i += kThreadsW) o[i] = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
      } else {
        float4* o = reinterpret_cast<float4*>(bT + h * N * 128 + p.nB * 32 * 128);
        for (int i = threadIdx.x; i < 32 * 128 / 16; i += kThreadsW) o[i] = make_float4(1.f, 1.f, 1.f, 1.f);
      }
    }
  }
  __syncthreads();
  // programmatic dependent launch: the set-up above overlapped the previous kernel's tail; from here on this
  // kernel reads / writes memory that kernel may have produced
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp == kConsumers / 32) {
    // =============================== TMA producer ===============================
    if (tile_begin < tile_end && ptx::elect_one()) {
      for (int i = 0; i < kMaxMaps; i++) ptx::prefetch_tmap(&p.maps[i]);
      uint32_t s = 0, ph = 0;
      int seg = tile_begin / p.ntiles, b = (tile_begin - seg * p.ntiles) / p.tiles_per_b;
      int tb = tile_begin - seg * p.ntiles - b * p.tiles_per_b;
      const int nA = 4 * p.nMB;
      for (int f = tile_begin; f < tile_end; f++) {
        const int t0 = tb * kTK;
        ptx::mbar_wait(&empty[s], ph ^ 1);
        ptx::mbar_arrive_expect_tx(&full[s], stage_bytes);
        unsigned char* st = ring + (size_t)s * stage_bytes;
        for (int i = 0; i < p.nops; i++) {
          const Op o = p.ops[i];
          int dst;
          if (o.dst_group >= nA) dst = 4 + o.dst_group - nA;                               // B operand
          else if (o.dst_group >= 4 * mb && o.dst_group < 4 * mb + 4) dst = o.dst_group - 4 * mb;   // this M-block's A
          else continue;
          const int cg = o.cgrp0 + (o.dst_group >= nA ? bcol0 >> 5 : 0) + seg * o.seg_cgrp_stride;
          const int t = t0 + ((o.flags & WG_SEG_SHIFT) ? p.seg_shift[seg] : o.shift);
          ptx::tma_load_4d(st + dst * kSub, &p.maps[o.map], &full[s], 0, t, cg, (o.flags & WG_LAYERED) ? seg * p.B + b : b);
        }
        if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
        if (++tb == p.tiles_per_b) {
          tb = 0;
          if (++b == p.B) { b = 0; seg++; }
        }
      }
    }
    return;
  }

  // =============================== consumers: transpose B, wgmma, flush ===============================
  const int wgi = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, tq = lane & 3;
  const int m0 = 64 * wgi + 16 * wq + g;          // A rows m0 and m0 + 8 of this thread's fragments
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; i++) d[i] = 0.f;
  auto write_slot = [&]() {   // this CTA's accumulator -> its scratch slot (every row and column, zeros included)
    float* slot = p.part + (size_t)blockIdx.x * 128 * N;
#pragma unroll
    for (int i = 0; i < N / 2; i += 2) {
      const int m = m0 + 8 * ((i >> 1) & 1), n = 8 * (i >> 2) + 2 * tq;
      *reinterpret_cast<float2*>(slot + (size_t)m * N + n) = make_float2(d[i], d[i + 1]);
    }
  };
  uint32_t s = 0, ph = 0;
  const int nvec = p.nB * 32 * 32 / 4;            // float4 pieces of the B sub-tiles
  // Stage i: B transposed into bT[i & 1], A fragments into register set i & 1, the ring stage released, then the MMAs of
  // stage i are issued and those of stage i - 1 waited for -- so the transpose of stage i + 1 overlaps the MMAs of stage i.
  // (wgmma reads its A registers asynchronously: the set of stage i is not touched again before stage i + 2.)
  if constexpr (BF16) {
    // as below with bf16 operands: each transpose step rounds two time rows of 4 channels into 4 bf16 pairs; the A
    // fragment of k16 step kk holds rows m, m + 8 at time rows 16 kk + 2 (lane % 4) (+ 8), each with its successor
    uint32_t a0[2][4], a1[2][4];
    const int nvec2 = p.nB * 32 * 32 / 8;
    auto stage = [&](uint32_t (&a)[2][4], unsigned char* bTh) {
      ptx::mbar_wait(&full[s], ph);
      const unsigned char* st = ring + (size_t)s * stage_bytes;
      ptx::named_bar(1, kConsumers);
      for (int idx = threadIdx.x; idx < nvec2; idx += kConsumers) {
        const int grp = idx >> 7, r = ((idx >> 3) & 15) * 2, c4 = idx & 7;   // B group, time row pair, 4-channel piece
        const unsigned char* src = st + (4 + grp) * kSub + ((c4 ^ (r & 7)) << 4);
        const float4 v0 = *reinterpret_cast<const float4*>(src + r * 128);
        const float4 v1 = *reinterpret_cast<const float4*>(st + (4 + grp) * kSub + (r + 1) * 128 + ((c4 ^ ((r + 1) & 7)) << 4));
        const float lo[4] = {v0.x, v0.y, v0.z, v0.w}, hi[4] = {v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int j = 0; j < 4; j++)
          *reinterpret_cast<uint32_t*>(bTh + ptx::sw64_off(grp * 32 + c4 * 4 + j, r)) = ptx::cvt_bf16x2(lo[j], hi[j]);
      }
#pragma unroll
      for (int kk = 0; kk < 2; kk++) {
#pragma unroll
        for (int h = 0; h < 4; h++) {
          const int m = m0 + 8 * (h & 1), kr = 16 * kk + 2 * tq + 8 * (h >> 1);
          const unsigned char* sub = st + (m >> 5) * kSub;
          a[kk][h] = ptx::cvt_bf16x2(*reinterpret_cast<const float*>(sub + ptx::sw128_off(kr, m & 31)),
                                     *reinterpret_cast<const float*>(sub + ptx::sw128_off(kr + 1, m & 31)));
        }
      }
      ptx::mbar_arrive(&empty[s]);
      if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
      ptx::fence_proxy_async();
      ptx::named_bar(1, kConsumers);
      ptx::wg_fence();
      const uint32_t b_u32 = ptx::smem_u32(bTh);
#pragma unroll
      for (int kk = 0; kk < 2; kk++) ptx::wgmma_rs_bf16<N>(d, a[kk], ptx::gmma_desc_k_sw64(b_u32 + 32 * kk), 1);
      ptx::wg_commit();
      ptx::wg_wait<1>();
    };
    for (int f = tile_begin; f < tile_end; f += 2) {
      stage(a0, bT);
      if (f + 1 < tile_end) stage(a1, bT + N * kBtRow);
    }
    ptx::wg_wait<0>();
    ptx::wg_touch(d);
    write_slot();
    return;
  }
  uint32_t a0[4][4], a1[4][4];
  auto stage = [&](uint32_t (&a)[4][4], unsigned char* bTh) {
    ptx::mbar_wait(&full[s], ph);
    const unsigned char* st = ring + (size_t)s * stage_bytes;
    ptx::named_bar(1, kConsumers);   // every consumer has waited for the MMAs of stage i - 2: bTh may be overwritten
    for (int idx = threadIdx.x; idx < nvec; idx += kConsumers) {
      const int grp = idx >> 8, r = (idx >> 3) & 31, c4 = idx & 7;   // B group, time row, 4-channel piece
      const float4 v = *reinterpret_cast<const float4*>(st + (4 + grp) * kSub + r * 128 + ((c4 ^ (r & 7)) << 4));
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int n = grp * 32 + c4 * 4 + j;
        *reinterpret_cast<float*>(bTh + ptx::sw128_off(n, r)) = vv[j];
      }
    }
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      const int k = 8 * kk + tq;
#pragma unroll
      for (int h = 0; h < 4; h++) {
        const int m = m0 + 8 * (h & 1), kr = k + 4 * (h >> 1);
        a[kk][h] = *reinterpret_cast<const uint32_t*>(st + (m >> 5) * kSub + ptx::sw128_off(kr, m & 31));
      }
    }
    ptx::mbar_arrive(&empty[s]);     // this thread's reads of the ring stage are done
    if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
    ptx::fence_proxy_async();
    ptx::named_bar(1, kConsumers);
    ptx::wg_fence();
    const uint32_t b_u32 = ptx::smem_u32(bTh);
#pragma unroll
    for (int kk = 0; kk < 4; kk++) ptx::wgmma_rs<N>(d, a[kk], ptx::gmma_desc_k_sw128(b_u32 + 32 * kk), 1);
    ptx::wg_commit();
    ptx::wg_wait<1>();
  };
  for (int f = tile_begin; f < tile_end; f += 2) {
    stage(a0, bT);
    if (f + 1 < tile_end) stage(a1, bT + N * 128);
  }
  ptx::wg_wait<0>();
  ptx::wg_touch(d);
  write_slot();
}

// C[seg][m][bcol0 + n] += sum over the ksplit slots of (M-block, column group, segment), in slot order; column 32 nB
// (the ones group) is the bias gradient db[seg][m] (column group 0 only)
__global__ void wgrad_reduce_kernel(const __grid_constant__ Params p) {
  const int nc = 32 * p.nB + p.use_ones;
  const int64_t total = (int64_t)p.nseg * p.n_split * p.nMB * 128 * nc;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = idx;
    const int n = (int)(r % nc); r /= nc;
    const int m = (int)(r % 128); r /= 128;
    const int mb = (int)(r % p.nMB); r /= p.nMB;
    const int ng = (int)(r % p.n_split);
    const int seg = (int)(r / p.n_split);
    if (m >= p.m_valid[mb]) continue;
    if (n >= 32 * p.nB && (ng != 0 || !p.db[mb])) continue;
    float sum = 0.f;
    for (int j = 0; j < p.ksplit; j++) {
      const int64_t slot = ((int64_t)(seg * p.ksplit + j) * p.n_split + ng) * p.nMB + mb;
      sum += p.part[(slot * 128 + m) * p.ncols + n];
    }
    if (n < 32 * p.nB) p.c[mb][(size_t)seg * p.c_seg_stride + (size_t)m * p.ldc + ng * 32 * p.nB + n] += sum;
    else p.db[mb][(size_t)seg * p.db_seg_stride + m] += sum;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// (B, T, C) fp32 channels-last tensor seen as {32 ch, T, C/32 groups, B} (the group axis OUTSIDE time, so that the box
// {32, 32, groups, 1} lands in shared memory group-major: `groups` consecutive [32 x 32] sub-tiles)
static bool make_act_map(CUtensorMap* m, const float* base, int C, int T, int B, int groups) {
  EncodeTiledFn enc = get_encode();
  if (!enc || C % 32 != 0) return false;
  cuuint64_t gdim[4] = {32, (cuuint64_t)T, (cuuint64_t)(C / 32), (cuuint64_t)B};
  cuuint64_t gstr[3] = {(cuuint64_t)C * 4, 128, (cuuint64_t)C * 4 * (cuuint64_t)T};
  cuuint32_t box[4] = {32, (cuuint32_t)kTK, (cuuint32_t)groups, 1}, es[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int N, bool BF16>
static cudaError_t launch_n(int grid, size_t smem, cudaStream_t st, const Params& p) {
  cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(wgrad_tc_kernel<N, BF16>), smem);
  if (e != cudaSuccess) return e;
  return launch_pdl(wgrad_tc_kernel<N, BF16>, grid, kThreadsW, smem, st, 1, p);
}

template <bool BF16>
static cudaError_t launch_bf(int N, int grid, size_t smem, cudaStream_t st, const Params& p) {
  switch (N) {
    case 32: return launch_n<32, BF16>(grid, smem, st, p);
    case 64: return launch_n<64, BF16>(grid, smem, st, p);
    case 96: return launch_n<96, BF16>(grid, smem, st, p);
    case 128: return launch_n<128, BF16>(grid, smem, st, p);
    case 160: return launch_n<160, BF16>(grid, smem, st, p);
    case 192: return launch_n<192, BF16>(grid, smem, st, p);
    case 224: return launch_n<224, BF16>(grid, smem, st, p);
    default: return launch_n<256, BF16>(grid, smem, st, p);
  }
}

}  // namespace wg

// For every block i:  C_i[128 x 32*sum(groups_b)] += A_i^T B   (+ db_i = column sums of A_i), one launch.
int wgrad_tc_blocks(const WgBlock* blocks, int nblocks, const WgOperand* b_ops, int nb_ops, int ldc, int B, int T,
                    cudaStream_t st, const WgOpts* opts) {
  using namespace wg;
  if (nblocks < 1 || nblocks > kMaxMB) { set_error("wgrad_tc: 1..%d M-blocks per launch", kMaxMB); return WNB_ERR_INVALID; }
  Params p;
  memset(&p, 0, sizeof(p));
  p.nMB = nblocks;
  p.nB = 0;
  for (int i = 0; i < nb_ops; i++) p.nB += b_ops[i].groups;
  bool any_db = false;
  for (int i = 0; i < nblocks; i++) any_db |= blocks[i].db != nullptr;
  p.use_ones = any_db ? 1 : 0;
  if (p.nB < 1 || p.nB > kMaxB - 1) { set_error("wgrad_tc: 1..7 B groups"); return WNB_ERR_INVALID; }
  const int N = 32 * (p.nB + p.use_ones);
  const bool bf16 = opts && opts->bf16;
  const int bt_bytes = 2 * N * (bf16 ? bt_row_bytes<true>() : bt_row_bytes<false>());   // the two transposed B tiles
  const int stage_bytes = (4 + p.nB) * kSub;
  int nst = (227 * 1024 - 1024 - 256 - bt_bytes) / stage_bytes;
  if (nst > 8) nst = 8;
  if (nst < 2) { set_error("wgrad_tc: stage too large"); return WNB_ERR_INVALID; }
  p.nstages = nst;

  int nmaps = 0;
  const float* map_base[kMaxMaps];
  int map_c[kMaxMaps], map_g[kMaxMaps];
  auto map_of = [&](const WgOperand& o) -> int {
    for (int i = 0; i < nmaps; i++)
      if (map_base[i] == o.base && map_c[i] == o.C && map_g[i] == o.groups) return i;
    if (nmaps >= kMaxMaps) return -1;
    const int nseg_map = (opts && opts->nseg > 1 && (o.flags & WG_LAYERED)) ? opts->nseg : 1;
    if (!make_act_map(&p.maps[nmaps], o.base, o.C, T, B * nseg_map, o.groups)) return -1;
    map_base[nmaps] = o.base; map_c[nmaps] = o.C; map_g[nmaps] = o.groups;
    return nmaps++;
  };
  auto add_op = [&](const WgOperand& o, int dst_group) -> bool {
    if (o.c0 % 32 != 0 || o.seg_cstride % 32 != 0 || o.groups < 1 || p.nops >= kMaxOps) return false;
    const int m = map_of(o);
    if (m < 0) return false;
    p.ops[p.nops++] = Op{m, o.c0 / 32, o.shift, o.flags, o.seg_cstride / 32, dst_group};
    return true;
  };
  for (int bi = 0; bi < nblocks; bi++) {
    int ng = 0;
    for (int i = 0; i < blocks[bi].nops; i++) {
      const WgOperand& o = blocks[bi].ops[i];
      if (ng + o.groups > 4) { set_error("wgrad_tc: more than 4 groups in an M-block"); return WNB_ERR_INVALID; }
      if (!add_op(o, bi * 4 + ng)) { set_error("wgrad_tc: tensor map creation failed (A)"); return WNB_ERR_CUDA; }
      ng += o.groups;
    }
    if (ng != 4) { set_error("wgrad_tc: an M-block needs exactly 4 groups"); return WNB_ERR_INVALID; }
    p.c[bi] = blocks[bi].c; p.m_valid[bi] = blocks[bi].m_valid; p.db[bi] = blocks[bi].db;
  }
  int nb = 0;
  for (int i = 0; i < nb_ops; i++) {
    if (!add_op(b_ops[i], 4 * nblocks + nb)) { set_error("wgrad_tc: tensor map creation failed (B)"); return WNB_ERR_CUDA; }
    nb += b_ops[i].groups;
  }
  for (int i = nmaps; i < kMaxMaps; i++) p.maps[i] = p.maps[0];
  p.ldc = ldc;
  p.n_split = (opts && opts->n_split > 1) ? opts->n_split : 1;
  p.nseg = (opts && opts->nseg > 1) ? opts->nseg : 1;
  if (p.nseg > 1 && (p.nseg > kMaxSeg || p.n_split > 1 || !opts->seg_shift)) {
    set_error("wgrad_tc: bad segment configuration (nseg=%d)", p.nseg);
    return WNB_ERR_INVALID;
  }
  // a WG_SEG_SHIFT operand takes its shift from the table also when there is one segment (a one-block stack)
  bool seg_shift_used = false;
  for (int i = 0; i < p.nops; i++) seg_shift_used |= (p.ops[i].flags & WG_SEG_SHIFT) != 0;
  if (seg_shift_used && !(opts && opts->seg_shift)) {
    set_error("wgrad_tc: a segment-shifted operand needs WgOpts::seg_shift");
    return WNB_ERR_INVALID;
  }
  if (opts && opts->seg_shift)
    for (int i = 0; i < p.nseg; i++) p.seg_shift[i] = opts->seg_shift[i];
  if (p.nseg > 1) {
    p.c_seg_stride = opts->c_seg_stride;
    p.db_seg_stride = opts->db_seg_stride;
  }
  p.T = T; p.B = B;
  p.tiles_per_b = (T + kTK - 1) / kTK;
  p.ntiles = B * p.tiles_per_b;
  const size_t smem = (size_t)bt_bytes + (size_t)nst * stage_bytes + 1024 + 256;
  const int sms = device_sms();
  const int sets = p.nMB * p.n_split * p.nseg;
  int ksplit = sms / sets;
  if (ksplit < 1) ksplit = 1;
  if (ksplit > p.ntiles) ksplit = p.ntiles;
  p.ksplit = ksplit;
  p.ncols = N;
  const int grid = sets * ksplit;
  p.part = static_cast<float*>(scratch_buffer(st, SCRATCH_WGRAD, (size_t)grid * 128 * N * sizeof(float)));
  if (!p.part) { set_error("wgrad_tc: cannot allocate the partial-sum scratch"); return WNB_ERR_CUDA; }
  const cudaError_t le = bf16 ? launch_bf<true>(N, grid, smem, st, p) : launch_bf<false>(N, grid, smem, st, p);
  if (le != cudaSuccess) { set_error("wgrad_tc: launch failed: %s", cudaGetErrorString(le)); return WNB_ERR_CUDA; }
  WNB_CHECK_LAUNCH("wgrad_tc");
  const int64_t total = (int64_t)p.nseg * p.n_split * p.nMB * 128 * (32 * p.nB + p.use_ones);
  const int64_t rblocks = (total + 255) / 256;
  wgrad_reduce_kernel<<<(int)(rblocks < sms * 8 ? rblocks : sms * 8), 256, 0, st>>>(p);
  WNB_CHECK_LAUNCH("wgrad_reduce");
  return WNB_OK;
}

// single M-block convenience wrapper
int wgrad_tc(const WgOperand* a_ops, int na_ops, const WgOperand* b_ops, int nb_ops, float* c, int ldc, int m_valid,
             float* db, int B, int T, cudaStream_t st) {
  if (na_ops < 1 || na_ops > 2) { set_error("wgrad_tc: 1 or 2 A operands"); return WNB_ERR_INVALID; }
  WgBlock blk;
  blk.nops = na_ops;
  for (int i = 0; i < na_ops; i++) blk.ops[i] = a_ops[i];
  blk.c = c; blk.m_valid = m_valid; blk.db = db;
  return wgrad_tc_blocks(&blk, 1, b_ops, nb_ops, ldc, B, T, st);
}

}  // namespace wnb
