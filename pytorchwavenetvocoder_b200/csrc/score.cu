// score.cu -- per-row cross entropy for held-out scoring (wnb_cross_entropy_rows, include/wnb200.h)
//
// wnb_cross_entropy partitions its sum over a grid that depends on B*T, so a row's share of the loss depends on what
// else is in the batch.  Here each row is summed in one fixed order that depends on that row alone:
//   * the value of position t is the float lse - logit[target] that wnb_cross_entropy computes for it (the Q == 256
//     register path when the logits are 16-byte aligned, the strided path otherwise: the same expressions, restated);
//   * positions are grouped in segments [32 j, 32 j + 32) of the row's own columns; lane i of a warp holds the value of
//     position 32 j + i (0 outside [start, length)) as a double, and the segment's sum is lane 0's result of an xor
//     butterfly over the 32 lanes;
//   * thread 0 of the row's first CTA adds the segment sums in ascending j to nll[b] (the caller zeroes it, or passes a previous window's sum).
// One cluster of CTAs per row, no atomics, and no dependence on the cluster or block size.  So a row's sum is
// bit-identical in any batch, with any padding, run after run; and a chain of calls over windows whose columns start at multiples of 32 (each
// scoring the positions after the previous window's) adds the same segment sums in the same order as one call over the
// whole row.
#include <cooperative_groups.h>

#include "common.cuh"

namespace wnb {

constexpr int kRowsThreads = 512;
constexpr int kSeg = 32;
constexpr int kCluster = 8;   // CTAs per row (the portable cluster size)
constexpr int kIlp = 4;       // positions whose loads a warp keeps in flight

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// cross_entropy_q256_kernel's value of one row (elementwise.cu), warp-uniform: a, b are the lane's columns
// 4 lane .. +3 and 128 + 4 lane .. +3 of the row lg, tg its target
__device__ __forceinline__ float ce_value_q256(float4 a, float4 b, const float* lg, int64_t tg) {
  float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  float m = v[0];
#pragma unroll
  for (int k = 1; k < 8; k++) m = fmaxf(m, v[k]);
  m = warp_max(m);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 8; k++) sum += expf(v[k] - m);
  sum = warp_sum(sum);
  const float lse = m + logf(sum);
  if (tg < 0 || tg >= 256) return NAN;
  return lse - lg[tg];
}

// cross_entropy_kernel's value of one row (elementwise.cu), warp-uniform
__device__ __forceinline__ float ce_value(const float* lg, int64_t tg, int Q, int lane) {
  float m = -INFINITY;
  for (int q = lane; q < Q; q += 32) m = fmaxf(m, lg[q]);
  m = warp_max(m);
  float s = 0.f;
  for (int q = lane; q < Q; q += 32) s += expf(lg[q] - m);
  s = warp_sum(s);
  const float lse = m + logf(s);
  if (tg < 0 || tg >= Q) return NAN;
  return lse - lg[tg];
}

// Rows are long and few (a 2^19-sample batch of 10 s utterances has three), so each row is a cluster of kCluster CTAs:
// in a round, warp w of CTA c takes segment jb + c * kWarps + w; after a cluster barrier, thread 0 of CTA 0 reads the
// round's segment sums from every CTA's shared memory (DSMEM) and adds them in ascending j.  The order is the same as one
// warp taking every segment in turn.  Within a segment a warp keeps kIlp positions' loads in flight.
template <bool kQ256>
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kRowsThreads, 1)
    cross_entropy_rows_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                              const int64_t* __restrict__ lengths, int start, double* __restrict__ nll,
                              int64_t* __restrict__ count, int T, int Q) {
  namespace cg = cooperative_groups;
  constexpr int kWarps = kRowsThreads / 32;
  __shared__ double seg_sum[kWarps];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x / kCluster;
  const int64_t len64 = lengths[b];
  const int len = (int)(len64 < 0 ? 0 : (len64 > T ? T : len64));
  if (len <= start) return;   // the same for every CTA of the cluster
  const int j0 = start / kSeg, j1 = (len + kSeg - 1) / kSeg;
  const float* lrow = logits + (size_t)b * T * Q;
  const int64_t* trow = target + (size_t)b * T;
  double acc = 0.0;
  if (rank == 0 && threadIdx.x == 0) acc = nll[b];
  for (int jb = j0; jb < j1; jb += kWarps * kCluster) {
    const int j = jb + rank * kWarps + warp;
    if (j < j1) {
      double mine = 0.0;
      const int p0 = j * kSeg;
      const int lo = p0 > start ? p0 : start, hi = p0 + kSeg < len ? p0 + kSeg : len;
      for (int pb = lo; pb < hi; pb += kIlp) {
        if (kQ256) {
          float4 a[kIlp], c[kIlp];
          int64_t tg[kIlp];
#pragma unroll
          for (int i = 0; i < kIlp; i++) {
            const int p = pb + i < hi ? pb + i : hi - 1;
            const float4* lg4 = reinterpret_cast<const float4*>(lrow + (size_t)p * Q);
            a[i] = lg4[lane];
            c[i] = lg4[32 + lane];
            tg[i] = trow[p];
          }
#pragma unroll
          for (int i = 0; i < kIlp; i++) {
            const int p = pb + i;
            const float v = ce_value_q256(a[i], c[i], lrow + (size_t)(p < hi ? p : hi - 1) * Q, tg[i]);
            if (p < hi && lane == p - p0) mine = (double)v;
          }
        } else {
#pragma unroll 1
          for (int p = pb; p < hi && p < pb + kIlp; p++) {
            const float v = ce_value(lrow + (size_t)p * Q, trow[p], Q, lane);
            if (lane == p - p0) mine = (double)v;
          }
        }
      }
      mine = warp_sum_f64(mine);
      if (lane == 0) seg_sum[warp] = mine;
    }
    cluster.sync();
    if (rank == 0 && threadIdx.x == 0) {
      for (int r = 0; r < kCluster; r++) {
        const double* part = cluster.map_shared_rank(seg_sum, r);
        const int jr = jb + r * kWarps;
        const int n = j1 - jr < kWarps ? j1 - jr : kWarps;
        for (int w = 0; w < n; w++) acc += part[w];
      }
    }
    cluster.sync();
  }
  if (rank == 0 && threadIdx.x == 0) {
    nll[b] = acc;
    if (count) count[b] += (int64_t)(len - start);
  }
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_cross_entropy_rows(const float* logits, const int64_t* target, const int64_t* lengths, int start,
                                   double* nll, int64_t* count, int B, int T, int Q, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && Q > 0 && start >= 0, "cross_entropy_rows: bad shape (B=%d T=%d Q=%d start=%d)", B, T, Q,
              start);
  WNB_REQUIRE(B <= (1 << 27), "cross_entropy_rows: B = %d rows is more than 2^27", B);
  WNB_REQUIRE(logits && target && lengths && nll, "cross_entropy_rows: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (Q == 256 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0)
    cross_entropy_rows_kernel<true><<<B * kCluster, kRowsThreads, 0, st>>>(logits, target, lengths, start, nll, count,
                                                                           T, Q);
  else
    cross_entropy_rows_kernel<false><<<B * kCluster, kRowsThreads, 0, st>>>(logits, target, lengths, start, nll, count,
                                                                            T, Q);
  WNB_CHECK_LAUNCH("cross_entropy_rows");
  return WNB_OK;
}

}  // extern "C"
