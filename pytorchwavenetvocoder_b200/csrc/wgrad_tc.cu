// wgrad_tc.cu -- tensor-core weight gradients:  C[m][n] += sum_{b,t} A[b][t][m] * Bm[b][t+shift][n]
//
// The reduction index is TIME.  With channels-last activations a TMA box [32 time rows x 32 channels] is an MN-major
// tile, and Hopper's tf32 wgmma takes K-major operands only.  So per 32-step stage the two consumer warpgroups
//   - transpose the B sub-tiles (up to 7 x 32 channels) into one K-major [N x 32] tile in shared memory, and
//   - read their A fragments (64 of the 128 M-block rows each) straight from the swizzled A sub-tiles into registers,
// then issue wgmma m64nNk8 (A from registers, B from shared memory; double-buffered, so the transpose of the next stage
// overlaps the MMAs of this one) into an fp32 accumulator that stays in registers for all the stages of one piece.
// A third role, one producer thread, streams the stages with TMA through an mbarrier ring.
//
// Work layout: one launch runs a LIST of problems.  A problem is one (M-block, column group, segment) of a call: a
// [128 x N] gradient summed over B x ceil(T/32) stages, cut into a fixed number of time chunks.  The host places the
// chunks of all problems on exactly one piece list per SM (wgrad_partition: static, from per-stage costs derived from
// the shapes), so a CTA may end one problem and start the next one, and problems of different N (one consumer loop
// instantiation each) share a launch.  Every chunk is summed from zero into its own slot of a scratch buffer;
// wgrad_reduce_kernel adds the slots of each problem into C in chunk order: no atomics, and the gradients depend
// neither on how the CTAs were scheduled nor on which CTA ran which chunk.
//
// Generic over "sub-tile lists": A = 4 groups of 32 channels (M = 128), B = up to 7 groups (N <= 224),
// each group = (tensor map, channel offset, time shift); dilated taps are just shifted groups, zero filled
// out of range by TMA.  An optional extra all-ones B group turns column 0 of that group into the bias
// gradient sum_t A[t][m] (replaces colsum_kernel).
// An M-block with at most 64 valid rows (dW2res at R = 64) loads only its 2 valid A sub-tiles, and only the first
// consumer warpgroup loads A fragments and issues wgmma: no load or MMA is spent on padding rows.
//
// bf16 operands (BF16 = true, WgOpts::bf16): the transpose writes B rounded to bf16 (cvt.rn.bf16x2 of two time rows)
// into a 64B-swizzled K-major [N x 32] bf16 tile, the A fragments are rounded the same way from the fp32 sub-tiles, and
// the MMAs are bf16 wgmma m64nNk16 with fp32 accumulation.  The all-ones rows are exact in bf16; slots and their
// reduction are unchanged.
#include <cuda.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/wnb200.h"
#include "common.cuh"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace wnb {
namespace wg {

constexpr int kMaxB = 8, kMaxMaps = 8, kMaxOps = 5;
constexpr int kMaxProb = 160, kMaxPieces = 448, kMaxCtas = 264;   // per launch (kernel parameters <= 32 KB)
constexpr int kConsumers = 256;              // two warpgroups: rows 0..63 and 64..127 of the M-block
constexpr int kThreadsW = kConsumers + 128;  // + the producer warpgroup (one thread issues TMA)
constexpr int kTK = 32;                      // time rows per stage (K of one stage)
constexpr int kSub = kTK * 128;              // one [32 x 32 fp32] swizzled sub-tile

// One TMA load per operand and stage: the tensor (B,T,C) is mapped 4-D as {32 ch, T, C/32 groups, B} with a box of
// {32, 32, groups, 1}, which lands in shared memory as `groups` consecutive [32 x 32] swizzled sub-tiles.  Everything
// per segment / column group is resolved on the host: channel group, time shift and batch offset.
struct Op { int16_t map, dst; int cgrp, shift, bofs; };
struct Prob {
  Op ops[kMaxOps];
  int8_t nops, nA, nB, ones;     // nA: A sub-tiles of a stage (4, or 2 for an M = 64 problem); ones: the all-ones group
  int ldc, m_valid;              // C rows m < m_valid, columns n < 32 nB
  float* c;
  float* db;                     // bias gradient (column 0 of the ones group) or null
  int16_t piece0, npieces;       // this problem's pieces: plist[piece0 ..], in the order the reduce adds them
};
struct Piece { int16_t prob; int s0, s1; int slot; };   // stages [s0, s1) of a problem; slot: float offset in `part`
struct alignas(64) Params {
  CUtensorMap maps[kMaxMaps];
  int T, B, tiles_per_b, nstages, stage_bytes, bt_half;   // stage_bytes: ring stage; bt_half: one transposed B tile
  float* part;
  int16_t cta_first[kMaxCtas + 1];   // CTA i runs pieces cta_first[i] .. cta_first[i + 1] - 1
  int16_t plist[kMaxPieces];
  Piece pieces[kMaxPieces];
  Prob probs[kMaxProb];
};
static_assert(sizeof(Params) <= 32000, "wgrad_tc: kernel parameters exceed the 32 KB limit");

// bytes of one row (32 time steps) of the transposed B tile
template <bool BF16>
__host__ __device__ constexpr int bt_row_bytes() { return BF16 ? 64 : 128; }

// The tf32 B transpose of one stage is cut into 64 nB units, each a 4 x 4 block of one B group: time rows 4 q .. 4 q + 3
// of channel chunk c4 (four 16-byte loads from the swizzled [32 x 32] sub-tile) become channels 4 c4 .. 4 c4 + 3 of time
// chunk q (four 16-byte stores into the K-major 128B-swizzled tile).  Unit u = 64 grp + 8 x + l has q = l, c4 = l ^ x:
// the 8 lanes of each quarter warp then load from 8 distinct 16-byte bank groups and store to 8 distinct ones, so every
// warp-wide load and store takes 4 shared-memory wavefronts for its 512 bytes.  (With c4 fixed per quarter warp the
// stores would still fill whole rows, but the loads of a quarter warp would hit only 2 bank groups.)
// Consumer thread t runs units t ^ 128, + 256, ...: warpgroup 1 takes the first ones, since in an M = 64 problem
// warpgroup 0 alone also loads the A fragments and issues the MMAs.
struct TrUnit { uint32_t src[4], dst[4]; };   // bytes from the first B sub-tile / from the transposed tile
__host__ __device__ __forceinline__ int tr_first_unit(int t) { return t ^ 128; }
__host__ __device__ __forceinline__ TrUnit tr_unit(int u) {
  const int grp = u >> 6, q = u & 7, c4 = q ^ ((u >> 3) & 7), r = 4 * q;
  TrUnit o;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    o.src[i] = grp * kSub + (r + i) * 128 + ((c4 ^ ((r + i) & 7)) << 4);   // time row r + i, channels 4 c4 ..
    o.dst[i] = ptx::sw128_off(grp * 32 + 4 * c4 + i, r);                  // channel 4 c4 + i, time rows r ..
  }
  return o;
}

// One piece with N = 32 (nB + ones): the consumer loop of both warpgroups.  Ring position (s, ph) carries over from
// piece to piece; the two transposed B tiles are free on entry (every wgmma of the previous piece has completed).
template <int N, bool BF16, bool M64>
__device__ __forceinline__ void run_piece(const Params& p, const Prob& pr, const Piece& pc, unsigned char* bT,
                                          const unsigned char* ring, uint64_t* full, uint64_t* empty, uint32_t& s,
                                          uint32_t& ph) {
  constexpr int kBtRow = bt_row_bytes<BF16>();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wgi = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, tq = lane & 3;
  constexpr int nA = M64 ? 2 : 4;
  const int ms = 64 * wgi + 16 * wq + g;          // slot rows ms and ms + 8 of this thread's accumulator fragments
  const int m0 = M64 ? ms - 64 * wgi : ms;        // A rows m0 and m0 + 8 (an M = 64 warpgroup covers rows 0..63)
  const int nB = pr.nB;
  ptx::named_bar(1, kConsumers);                 // both warpgroups are past the previous piece's last wgmma
  if (pr.ones) {   // the ones rows of both transposed B tiles (32 rows after the nB * 32 transposed ones)
    for (int h = 0; h < 2; h++) {
      if constexpr (BF16) {
        uint4* o = reinterpret_cast<uint4*>(bT + h * N * kBtRow + nB * 32 * kBtRow);
        for (int i = threadIdx.x; i < 32 * kBtRow / 16; i += kConsumers) o[i] = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
      } else {
        float4* o = reinterpret_cast<float4*>(bT + h * N * 128 + nB * 32 * 128);
        for (int i = threadIdx.x; i < 32 * 128 / 16; i += kConsumers) o[i] = make_float4(1.f, 1.f, 1.f, 1.f);
      }
    }
  }
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; i++) d[i] = 0.f;
  // Stage i: B transposed into bT[i & 1], A fragments into register set i & 1, the ring stage released, then the MMAs of
  // stage i are issued and those of stage i - 1 waited for -- so the transpose of stage i + 1 overlaps the MMAs of stage i.
  // (wgmma reads its A registers asynchronously: the set of stage i is not touched again before stage i + 2.)
  // M = 64: warpgroup 0 issues every stage's MMAs for rows 0..63 (the same wgmma sequence the M = 128 form issues for
  // them, so the sums are the same); warpgroup 1 only shares the transposes.
  if constexpr (BF16) {
    // as below with bf16 operands: each transpose step rounds two time rows of 4 channels into 4 bf16 pairs; the A
    // fragment of k16 step kk holds rows m, m + 8 at time rows 16 kk + 2 (lane % 4) (+ 8), each with its successor
    uint32_t a0[2][4], a1[2][4];
    const int nvec2 = nB * 32 * 32 / 8;
    auto stage = [&](uint32_t (&a)[2][4], unsigned char* bTh, bool mine) {
      ptx::mbar_wait(&full[s], ph);
      const unsigned char* st = ring + (size_t)s * p.stage_bytes;
      ptx::named_bar(1, kConsumers);
      for (int idx = threadIdx.x; idx < nvec2; idx += kConsumers) {
        const int grp = idx >> 7, r = ((idx >> 3) & 15) * 2, c4 = idx & 7;   // B group, time row pair, 4-channel piece
        const unsigned char* src = st + (nA + grp) * kSub + ((c4 ^ (r & 7)) << 4);
        const float4 v0 = *reinterpret_cast<const float4*>(src + r * 128);
        const float4 v1 = *reinterpret_cast<const float4*>(st + (nA + grp) * kSub + (r + 1) * 128 + ((c4 ^ ((r + 1) & 7)) << 4));
        const float lo[4] = {v0.x, v0.y, v0.z, v0.w}, hi[4] = {v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int j = 0; j < 4; j++)
          *reinterpret_cast<uint32_t*>(bTh + ptx::sw64_off(grp * 32 + c4 * 4 + j, r)) = ptx::cvt_bf16x2(lo[j], hi[j]);
      }
      if (mine) {
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
      }
      ptx::mbar_arrive(&empty[s]);
      if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
      ptx::fence_proxy_async();
      ptx::named_bar(1, kConsumers);
      if (mine) {
        ptx::wg_fence();
        const uint32_t b_u32 = ptx::smem_u32(bTh);
#pragma unroll
        for (int kk = 0; kk < 2; kk++) ptx::wgmma_rs_bf16<N>(d, a[kk], ptx::gmma_desc_k_sw64(b_u32 + 32 * kk), 1);
        ptx::wg_commit();
        ptx::wg_wait<1>();
      } else {
        ptx::wg_wait<0>();
      }
    };
    for (int f = pc.s0; f < pc.s1; f += 2) {
      stage(a0, bT, !M64 || wgi == 0);
      if (f + 1 < pc.s1) stage(a1, bT + N * kBtRow, !M64 || wgi == 0);
    }
  } else {
    uint32_t a0[4][4], a1[4][4];
    const int nunit = nB * 64;                    // 4 x 4 transpose units of the B sub-tiles (tr_unit)
    auto stage = [&](uint32_t (&a)[4][4], unsigned char* bTh, bool mine) {
      ptx::mbar_wait(&full[s], ph);
      const unsigned char* st = ring + (size_t)s * p.stage_bytes;
      const unsigned char* sB = st + nA * kSub;
      ptx::named_bar(1, kConsumers);   // every consumer has waited for the MMAs of stage i - 2: bTh may be overwritten
      for (int u = tr_first_unit(threadIdx.x); u < nunit; u += kConsumers) {
        const TrUnit o = tr_unit(u);
        float4 v[4];
#pragma unroll
        for (int i = 0; i < 4; i++) v[i] = *reinterpret_cast<const float4*>(sB + o.src[i]);
        *reinterpret_cast<float4*>(bTh + o.dst[0]) = make_float4(v[0].x, v[1].x, v[2].x, v[3].x);
        *reinterpret_cast<float4*>(bTh + o.dst[1]) = make_float4(v[0].y, v[1].y, v[2].y, v[3].y);
        *reinterpret_cast<float4*>(bTh + o.dst[2]) = make_float4(v[0].z, v[1].z, v[2].z, v[3].z);
        *reinterpret_cast<float4*>(bTh + o.dst[3]) = make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
      }
      if (mine) {
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
          const int k = 8 * kk + tq;
#pragma unroll
          for (int h = 0; h < 4; h++) {
            const int m = m0 + 8 * (h & 1), kr = k + 4 * (h >> 1);
            a[kk][h] = *reinterpret_cast<const uint32_t*>(st + (m >> 5) * kSub + ptx::sw128_off(kr, m & 31));
          }
        }
      }
      ptx::mbar_arrive(&empty[s]);     // this thread's reads of the ring stage are done
      if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
      ptx::fence_proxy_async();
      ptx::named_bar(1, kConsumers);
      if (mine) {
        ptx::wg_fence();
        const uint32_t b_u32 = ptx::smem_u32(bTh);
#pragma unroll
        for (int kk = 0; kk < 4; kk++) ptx::wgmma_rs<N>(d, a[kk], ptx::gmma_desc_k_sw128(b_u32 + 32 * kk), 1);
        ptx::wg_commit();
        ptx::wg_wait<1>();
      } else {
        ptx::wg_wait<0>();
      }
    };
    for (int f = pc.s0; f < pc.s1; f += 2) {
      stage(a0, bT, !M64 || wgi == 0);
      if (f + 1 < pc.s1) stage(a1, bT + N * 128, !M64 || wgi == 0);
    }
  }
  ptx::wg_wait<0>();
  ptx::wg_touch(d);
  // the accumulator -> this piece's slot (every row and column, zeros included; M = 64: rows 0..63)
  if (M64 && wgi == 1) return;
  float* slot = p.part + pc.slot;
#pragma unroll
  for (int i = 0; i < N / 2; i += 2) {
    const int m = ms + 8 * ((i >> 1) & 1), n = 8 * (i >> 2) + 2 * tq;
    *reinterpret_cast<float2*>(slot + (size_t)m * N + n) = make_float2(d[i], d[i + 1]);
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kThreadsW, 1) wgrad_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ unsigned char smem_raw[];
  // aligned by pointer arithmetic on smem_raw (not through an integer), so that the compiler still knows every pointer
  // derived from it is a shared-memory one and emits LDS / STS instead of generic loads and stores
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* bT = smem;                                   // 2 x K-major [N x 32] B tile (+ the ones rows)
  unsigned char* ring = smem + 2 * p.bt_half;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)p.nstages * p.stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.nstages;
  const int warp = threadIdx.x >> 5;
  const int pc0 = p.cta_first[blockIdx.x], pc1 = p.cta_first[blockIdx.x + 1];

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kConsumers);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch: the set-up above overlapped the previous kernel's tail; from here on this
  // kernel reads / writes memory that kernel may have produced
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  if (pc0 == pc1) return;   // a CTA without work (fewer stages than SMs)

  if (warp >= kConsumers / 32) {
    // =============================== TMA producer warpgroup ===============================
    // setmaxnreg hands the producer's registers to the consumers (232 each: N = 256 holds 128 accumulator registers)
    ptx::setmaxnreg_dec<40>();
    if (warp == kConsumers / 32 && ptx::elect_one()) {
      for (int i = 0; i < kMaxMaps; i++) ptx::prefetch_tmap(&p.maps[i]);
      uint32_t s = 0, ph = 0;
      for (int q = pc0; q < pc1; q++) {
        const Piece& pc = p.pieces[q];
        const Prob& pr = p.probs[pc.prob];
        const int bytes = (pr.nA + pr.nB) * kSub;
        int b = pc.s0 / p.tiles_per_b, tb = pc.s0 - b * p.tiles_per_b;
        for (int f = pc.s0; f < pc.s1; f++) {
          const int t0 = tb * kTK;
          ptx::mbar_wait(&empty[s], ph ^ 1);
          ptx::mbar_arrive_expect_tx(&full[s], bytes);
          unsigned char* st = ring + (size_t)s * p.stage_bytes;
          for (int i = 0; i < pr.nops; i++) {
            const Op& o = pr.ops[i];
            ptx::tma_load_4d(st + o.dst * kSub, &p.maps[o.map], &full[s], 0, t0 + o.shift, o.cgrp, o.bofs + b);
          }
          if (++s == (uint32_t)p.nstages) { s = 0; ph ^= 1; }
          if (++tb == p.tiles_per_b) { tb = 0; b++; }
        }
      }
    }
    return;
  }

  // =============================== consumers: transpose B, wgmma, flush ===============================
  ptx::setmaxnreg_inc<232>();
  uint32_t s = 0, ph = 0;
  for (int q = pc0; q < pc1; q++) {
    const Piece& pc = p.pieces[q];
    const Prob& pr = p.probs[pc.prob];
    const int N = 32 * (pr.nB + pr.ones);
    if (pr.nA == 2) {   // M = 64 (problems with N <= 128 only, see wgrad_tc_multi)
      switch (N) {
        case 32: run_piece<32, BF16, true>(p, pr, pc, bT, ring, full, empty, s, ph); break;
        case 64: run_piece<64, BF16, true>(p, pr, pc, bT, ring, full, empty, s, ph); break;
        case 96: run_piece<96, BF16, true>(p, pr, pc, bT, ring, full, empty, s, ph); break;
        default: run_piece<128, BF16, true>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      }
      continue;
    }
    switch (N) {
      case 32: run_piece<32, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 64: run_piece<64, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 96: run_piece<96, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 128: run_piece<128, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 160: run_piece<160, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 192: run_piece<192, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      case 224: run_piece<224, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
      default: run_piece<256, BF16, false>(p, pr, pc, bT, ring, full, empty, s, ph); break;
    }
  }
}

// C[m][n] += sum over the problem's pieces of their slots, in piece order (problem = blockIdx.y); column 32 nB (the
// ones group) is the bias gradient db[m].
__global__ void wgrad_reduce_kernel(const __grid_constant__ Params p) {
  const Prob& pr = p.probs[blockIdx.y];
  if (pr.npieces == 0) return;
  const int N = 32 * (pr.nB + pr.ones), nc = 32 * pr.nB + (pr.db ? 1 : 0);
  const int total = pr.m_valid * nc;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int m = idx / nc, n = idx - m * nc;
    float sum = 0.f;
    for (int j = 0; j < pr.npieces; j++) {
      const float* sl = p.part + p.pieces[p.plist[pr.piece0 + j]].slot + (size_t)m * N + n;
      sum += sl[0];
    }
    if (n < 32 * pr.nB) pr.c[(size_t)m * pr.ldc + n] += sum;
    else pr.db[m] += sum;
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

template <bool BF16>
static cudaError_t launch(int grid, size_t smem, cudaStream_t st, const Params& p) {
  cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(wgrad_tc_kernel<BF16>), smem);
  if (e != cudaSuccess) return e;
  return launch_pdl(wgrad_tc_kernel<BF16>, grid, kThreadsW, smem, st, 1, p);
}

// Time of one stage on one SM (microseconds), from the problem's shape: the larger of streaming its HBM bytes through
// the CTA's ring and the work of the consumer warpgroups (B transpose and A fragment loads per element, wgmma per
// flop at the dense tf32 rate of one SM, 3.75 TFLOP/s).  The per-element and streaming constants are fitted to the
// per-piece times of this kernel's tf32 path (the 4 x 4 register-block transpose) measured with %globaltimer on an
// H100 80GB HBM3 (700 W power limit, SM clock 1980 MHz) at the bench shape: dWskip 0.89 us per stage (N = 224,
// 6 transposed groups), dW1 0.85 (N = 192, 5 groups), 0.73 for N = 160 with 4 groups, all consumer-bound (the
// B-element constant is their least-squares fit), and dW2res 0.50 (16 KB per stage streamed, ~33 GB/s per SM with four
// ring stages in flight).
static double stage_cost_us(int M, int N, int nB, double hbm_bytes, bool bf16) {
  const double stream_us = hbm_bytes / 32.8e3;
  const double flop_us = 2.0 * M * N * kTK / (bf16 ? 7.5e6 : 3.75e6);
  const double elem_us = 6.4e-5 * nB * 32.0 * kTK + 1.6e-5 * (double)M * kTK;
  return fmax(stream_us, flop_us + elem_us);
}

}  // namespace wg

// Static partition of a problem list over `sms` CTAs (see tc_host.h).  Problem i is cut into nchunk[i] time chunks of
// ceil(stages / nchunk) stages; a chunk is the unit of work: one CTA sums it from zero in its registers and writes it to
// one slot, and the reduce adds a problem's chunks in chunk order.  The chunks therefore fix the summation order, and
// the placement below only decides which CTA runs which chunk, and when.
// Problems with lock[i] != 0 share operands through L2 and must stream the same time range at the same time: chunk c of
// locked problem i goes to CTA c * nlocked + i, so all CTAs of one chunk start together.  The other chunks go, longest
// first, to the CTA with the least cost so far.  CTAs of odd locked chunks run those chunks first, the others after
// their locked chunk, so that streaming-bound stages run beside the locked ones all the time.
int wgrad_partition(const int* stages, const int* nchunk, const double* cost, const int* lock, int nprob, int sms,
                    int* cta_first, WgPiece* pieces, int max_pieces) {
  if (nprob < 0 || sms < 1 || !cta_first || (nprob > 0 && (!stages || !nchunk || !cost || !lock))) return -1;
  std::vector<int> locked;
  for (int i = 0; i < nprob; i++) {
    if (stages[i] < 0 || nchunk[i] < 1 || !(cost[i] >= 0.0)) return -1;
    if (stages[i] > 0 && lock[i]) locked.push_back(i);
  }
  auto chunk = [&](int i, int c, int& s0, int& s1) {
    const int per = (stages[i] + nchunk[i] - 1) / nchunk[i];
    s0 = (int)std::min<int64_t>(stages[i], (int64_t)c * per);
    s1 = (int)std::min<int64_t>(stages[i], (int64_t)(c + 1) * per);
  };
  const int nl = (int)locked.size();
  bool place_locked = nl > 0;
  for (int i : locked) place_locked &= nchunk[i] == nchunk[locked[0]];
  if (place_locked && (int64_t)nl * nchunk[locked[0]] > sms) place_locked = false;
  std::vector<double> load(sms, 0.0);
  std::vector<WgPiece> own(sms, WgPiece{-1, 0, 0});   // each CTA's locked chunk
  std::vector<std::vector<WgPiece>> rest(sms);
  struct Unit { double w; int prob, s0, s1; };
  std::vector<Unit> units;
  for (int i = 0; i < nprob; i++) {
    if (stages[i] == 0) continue;
    const bool mine = place_locked && lock[i];
    const int li = mine ? (int)(std::find(locked.begin(), locked.end(), i) - locked.begin()) : 0;
    for (int c = 0; c < nchunk[i]; c++) {
      int s0, s1;
      chunk(i, c, s0, s1);
      if (s1 <= s0) continue;
      if (mine) {
        const int j = c * nl + li;
        own[j] = WgPiece{i, s0, s1};
        load[j] += (s1 - s0) * cost[i];
      } else {
        units.push_back(Unit{(s1 - s0) * cost[i], i, s0, s1});
      }
    }
  }
  std::stable_sort(units.begin(), units.end(), [](const Unit& a, const Unit& b) { return a.w > b.w; });
  for (const Unit& u : units) {
    int j = 0;
    for (int t = 1; t < sms; t++)
      if (load[t] < load[j]) j = t;
    load[j] += u.w;
    rest[j].push_back(WgPiece{u.prob, u.s0, u.s1});
  }
  int np = 0;
  auto emit = [&](const WgPiece& w) -> bool {
    if (pieces && np >= max_pieces) return false;
    if (pieces) pieces[np] = w;
    np++;
    return true;
  };
  for (int j = 0; j < sms; j++) {
    cta_first[j] = np;
    const bool rest_first = own[j].prob >= 0 && ((j / nl) & 1);
    if (rest_first)
      for (const WgPiece& w : rest[j])
        if (!emit(w)) return -1;
    if (own[j].prob >= 0 && !emit(own[j])) return -1;
    if (!rest_first)
      for (const WgPiece& w : rest[j])
        if (!emit(w)) return -1;
  }
  cta_first[sms] = np;
  return np;
}

// Every call's C_i[128 x 32*sum(groups_b)] += A_i^T B (+ db_i = column sums of A_i) for all its M-blocks, column groups
// and segments: one problem list, one launch of device_sms() CTAs and one reduce (more only if the list exceeds the
// kernel's parameter tables).
int wgrad_tc_multi(const WgCall* calls, int ncalls, int B, int T, cudaStream_t st) {
  using namespace wg;
  if (ncalls < 1 || B < 1 || T < 1) { set_error("wgrad_tc: bad call list"); return WNB_ERR_INVALID; }
  const bool bf16 = calls[0].opts.bf16 != 0;
  const int sms = device_sms() < kMaxCtas ? device_sms() : kMaxCtas;
  const int tiles_per_b = (T + kTK - 1) / kTK, ntiles = B * tiles_per_b;

  static thread_local Params p;   // ~30 KB: kept off the call stack
  memset(&p, 0, sizeof(p));
  int nmaps = 0;
  const float* map_base[kMaxMaps];
  int map_c[kMaxMaps], map_g[kMaxMaps], map_b[kMaxMaps];
  auto map_of = [&](const float* base, int C, int groups, int nbatch) -> int {
    for (int i = 0; i < nmaps; i++)
      if (map_base[i] == base && map_c[i] == C && map_g[i] == groups && map_b[i] == nbatch) return i;
    if (nmaps >= kMaxMaps) return -1;
    if (!make_act_map(&p.maps[nmaps], base, C, T, nbatch, groups)) return -1;
    map_base[nmaps] = base; map_c[nmaps] = C; map_g[nmaps] = groups; map_b[nmaps] = nbatch;
    return nmaps++;
  };

  std::vector<Prob> probs;
  std::vector<double> cost;
  std::vector<int> lock, chunks;
  int maxN = 32, max_stage = 0;
  for (int ci = 0; ci < ncalls; ci++) {
    const WgCall& cl = calls[ci];
    const WgOpts& o = cl.opts;
    if ((o.bf16 != 0) != bf16) { set_error("wgrad_tc: tf32 and bf16 calls in one list"); return WNB_ERR_INVALID; }
    if (cl.nblocks < 1 || cl.nblocks > 5) { set_error("wgrad_tc: 1..5 M-blocks per call"); return WNB_ERR_INVALID; }
    int nB = 0;
    for (int i = 0; i < cl.nb_ops; i++) nB += cl.b_ops[i].groups;
    if (nB < 1 || nB > kMaxB - 1) { set_error("wgrad_tc: 1..7 B groups"); return WNB_ERR_INVALID; }
    bool any_db = false;
    for (int i = 0; i < cl.nblocks; i++) any_db |= cl.blocks[i].db != nullptr;
    const int ones = any_db ? 1 : 0, N = 32 * (nB + ones);
    const int n_split = o.n_split > 1 ? o.n_split : 1, nseg = o.nseg > 1 ? o.nseg : 1;
    if (nseg > 1 && n_split > 1) { set_error("wgrad_tc: segments and column groups in one call"); return WNB_ERR_INVALID; }
    bool seg_shift_used = false;
    for (int i = 0; i < cl.nb_ops; i++) seg_shift_used |= (cl.b_ops[i].flags & WG_SEG_SHIFT) != 0;
    for (int bi = 0; bi < cl.nblocks; bi++)
      for (int i = 0; i < cl.blocks[bi].nops; i++) seg_shift_used |= (cl.blocks[bi].ops[i].flags & WG_SEG_SHIFT) != 0;
    if (seg_shift_used && !o.seg_shift) {
      set_error("wgrad_tc: a segment-shifted operand needs WgOpts::seg_shift");
      return WNB_ERR_INVALID;
    }
    const bool locked = cl.nblocks * n_split > 1;   // operands shared through L2 by several problems of this call
    // time chunks per problem: the SMs shared evenly by the call's problems (at least one chunk, at most one per
    // stage).  A chunk is summed by one CTA from zero, so this fixes the summation order of the call's gradients.
    int k = device_sms() / (cl.nblocks * n_split * nseg);
    k = k < 1 ? 1 : (k > ntiles ? ntiles : k);
    maxN = N > maxN ? N : maxN;
    for (int seg = 0; seg < nseg; seg++)
      for (int ng = 0; ng < n_split; ng++)
        for (int bi = 0; bi < cl.nblocks; bi++) {
          const WgBlock& blk = cl.blocks[bi];
          Prob pr;
          memset(&pr, 0, sizeof(pr));
          pr.nA = (blk.m_valid <= 64 && N <= 128) ? 2 : 4;
          pr.nB = (int8_t)nB;
          pr.ones = (int8_t)ones;
          double bytes = 0.0;
          auto add_op = [&](const WgOperand& w, int dst, int groups, double share) -> bool {
            if (w.c0 % 32 != 0 || w.seg_cstride % 32 != 0 || w.groups < 1 || pr.nops >= kMaxOps) return false;
            const bool layered = (w.flags & WG_LAYERED) != 0;
            const int m = map_of(w.base, w.C, groups, layered ? B * nseg : B);
            if (m < 0) return false;
            const int cgrp = w.c0 / 32 + seg * (w.seg_cstride / 32) + (dst >= pr.nA ? ng * nB : 0);
            const int shift = (w.flags & WG_SEG_SHIFT) ? o.seg_shift[seg] : w.shift;
            bool dup = false;   // another tap of the same channels (a dilated copy): read from L2
            for (int i = 0; i < pr.nops; i++) dup |= pr.ops[i].map == m && pr.ops[i].cgrp == cgrp;
            const bool same_per_seg = !layered && w.seg_cstride == 0 && !(w.flags & WG_SEG_SHIFT);   // aux of dW1
            if (!dup) bytes += groups * (double)kSub / (nseg > 1 && same_per_seg ? nseg : share);
            pr.ops[pr.nops++] = Op{(int16_t)m, (int16_t)dst, cgrp, shift, layered ? seg * B : 0};
            return true;
          };
          int na = 0;
          for (int i = 0; i < blk.nops; i++) {
            const WgOperand& w = blk.ops[i];
            if (na + w.groups > 4) { set_error("wgrad_tc: more than 4 groups in an M-block"); return WNB_ERR_INVALID; }
            const int keep = pr.nA - na < w.groups ? pr.nA - na : w.groups;   // M = 64: rows >= 64 are not loaded
            if (keep > 0 && !add_op(w, na, keep, locked ? n_split : 1)) {
              set_error("wgrad_tc: tensor map creation failed (A)");
              return WNB_ERR_CUDA;
            }
            na += w.groups;
          }
          if (na != 4) { set_error("wgrad_tc: an M-block needs exactly 4 groups"); return WNB_ERR_INVALID; }
          int nb = 0;
          for (int i = 0; i < cl.nb_ops; i++) {
            if (!add_op(cl.b_ops[i], pr.nA + nb, cl.b_ops[i].groups, locked ? cl.nblocks : 1)) {
              set_error("wgrad_tc: tensor map creation failed (B)");
              return WNB_ERR_CUDA;
            }
            nb += cl.b_ops[i].groups;
          }
          pr.ldc = cl.ldc;
          pr.m_valid = blk.m_valid;
          pr.c = blk.c + (size_t)seg * o.c_seg_stride + ng * 32 * nB;
          pr.db = (ng == 0 && blk.db) ? blk.db + (size_t)seg * o.db_seg_stride : nullptr;
          const int stage_bytes = (pr.nA + nB) * kSub;
          max_stage = stage_bytes > max_stage ? stage_bytes : max_stage;
          probs.push_back(pr);
          cost.push_back(stage_cost_us(32 * pr.nA, N, nB, bytes, bf16));
          lock.push_back(locked ? 1 : 0);
          chunks.push_back(k);
        }
  }
  for (int i = nmaps; i < kMaxMaps; i++) p.maps[i] = p.maps[0];

  const int bt_half = maxN * (bf16 ? bt_row_bytes<true>() : bt_row_bytes<false>());
  int nst = (227 * 1024 - 1024 - 256 - 2 * bt_half) / max_stage;
  if (nst > 8) nst = 8;
  if (nst < 2) { set_error("wgrad_tc: stage too large"); return WNB_ERR_INVALID; }
  const size_t smem = (size_t)2 * bt_half + (size_t)nst * max_stage + 1024 + 256;
  p.T = T; p.B = B; p.tiles_per_b = tiles_per_b;
  p.nstages = nst; p.stage_bytes = max_stage; p.bt_half = bt_half;

  std::vector<int> stages;
  std::vector<int> cta_first(sms + 1);
  std::vector<WgPiece> pcs(kMaxPieces);
  for (size_t p0 = 0; p0 < probs.size(); p0 += kMaxProb) {
    const int n = (int)(probs.size() - p0 < (size_t)kMaxProb ? probs.size() - p0 : kMaxProb);
    stages.assign(n, ntiles);
    const int np = wgrad_partition(stages.data(), chunks.data() + p0, cost.data() + p0, lock.data() + p0, n, sms,
                                   cta_first.data(), pcs.data(), kMaxPieces);
    if (np < 0) { set_error("wgrad_tc: more than %d pieces", kMaxPieces); return WNB_ERR_INVALID; }
    for (int i = 0; i <= sms; i++) p.cta_first[i] = (int16_t)cta_first[i];
    size_t slots = 0;
    for (int i = 0; i < n; i++) {
      p.probs[i] = probs[p0 + i];
      p.probs[i].npieces = 0;
    }
    for (int q = 0; q < np; q++) {
      const Prob& pr = p.probs[pcs[q].prob];
      p.pieces[q] = Piece{(int16_t)pcs[q].prob, pcs[q].s0, pcs[q].s1, (int)slots};
      slots += (size_t)128 * 32 * (pr.nB + pr.ones);
    }
    int k = 0;
    for (int i = 0; i < n; i++) {   // each problem's chunks in time order: the order its slots are added in
      p.probs[i].piece0 = (int16_t)k;
      for (int q = 0; q < np; q++)
        if (pcs[q].prob == i) { p.plist[k++] = (int16_t)q; p.probs[i].npieces++; }
      std::sort(p.plist + p.probs[i].piece0, p.plist + k,
                [&](int16_t a, int16_t b) { return pcs[a].s0 < pcs[b].s0; });
    }
    if (slots > (size_t)INT32_MAX) { set_error("wgrad_tc: partial-sum scratch too large"); return WNB_ERR_INVALID; }
    p.part = static_cast<float*>(scratch_buffer(st, SCRATCH_WGRAD, (slots ? slots : 1) * sizeof(float)));
    if (!p.part) { set_error("wgrad_tc: cannot allocate the partial-sum scratch"); return WNB_ERR_CUDA; }
    const cudaError_t le = bf16 ? launch<true>(sms, smem, st, p) : launch<false>(sms, smem, st, p);
    if (le != cudaSuccess) { set_error("wgrad_tc: launch failed: %s", cudaGetErrorString(le)); return WNB_ERR_CUDA; }
    WNB_CHECK_LAUNCH("wgrad_tc");
    int gx = (sms * 8 + n - 1) / n;
    if (gx > 64) gx = 64;
    wgrad_reduce_kernel<<<dim3(gx, n), 256, 0, st>>>(p);
    WNB_CHECK_LAUNCH("wgrad_reduce");
  }
  return WNB_OK;
}

int wgrad_tc_blocks(const WgBlock* blocks, int nblocks, const WgOperand* b_ops, int nb_ops, int ldc, int B, int T,
                    cudaStream_t st, const WgOpts* opts) {
  WgCall c;
  memset(&c, 0, sizeof(c));
  c.blocks = blocks; c.nblocks = nblocks; c.b_ops = b_ops; c.nb_ops = nb_ops; c.ldc = ldc;
  if (opts) c.opts = *opts;
  return wgrad_tc_multi(&c, 1, B, T, st);
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

WNB_API int wnb_wgrad_partition(const int* stages, const int* nchunk, const double* cost, const int* lock, int nprob,
                                int sms, int* cta_first, int* pieces, int max_pieces) {
  static_assert(sizeof(wnb::WgPiece) == 3 * sizeof(int), "WgPiece is three ints");
  const int np = wnb::wgrad_partition(stages, nchunk, cost, lock, nprob, sms, cta_first,
                                      reinterpret_cast<wnb::WgPiece*>(pieces), max_pieces);
  if (np < 0) wnb::set_error("wgrad_partition: bad arguments or more than %d pieces", max_pieces);
  return np < 0 ? WNB_ERR_INVALID : np;
}

WNB_API int wnb_wgrad_transpose_map(int nB, int* map) {
  using namespace wnb::wg;
  if (nB < 1 || nB > kMaxB - 1 || !map) {
    wnb::set_error("wgrad_transpose_map: 1..7 B groups and a map");
    return WNB_ERR_INVALID;
  }
  int k = 0;
  for (int t = 0; t < kConsumers; t++)   // the consumer loop of run_piece, thread by thread
    for (int u = tr_first_unit(t), it = 0; u < nB * 64; u += kConsumers, it++) {
      const TrUnit o = tr_unit(u);
      int* row = map + 10 * k++;
      row[0] = t; row[1] = it;
      for (int i = 0; i < 4; i++) { row[2 + i] = (int)o.src[i]; row[6 + i] = (int)o.dst[i]; }
    }
  return k;
}
