// distortion.cu -- mel-cepstral distortion between two lists of mel-cepstra (wnb_mcd_aligned, wnb_mcd_dtw,
// include/wnb200.h), float64 with explicit round-to-nearest operations (nothing is contracted to FMA), fixed orders, no
// atomics: a pair gives the same bits alone or in any batch, run after run.
//
// Local distance of frames a, b (columns 1 .. D; c0 is column 0 and is left out): dist = sqrt(s),
// s = sum_{d=1..D} (a_d - b_d)^2 added in ascending d.
//
// wnb_mcd_aligned: one CTA per pair (grid-stride).  Frames t < n = min(Tr, Td) are compared index by index.  Lane l of a
// warp holds dist of frame 32 c + l of chunk c (0.0 past n); the chunk's sum is lane 0's value after an xor butterfly
// (v += v[l ^ o] for o = 16, 8, 4, 2, 1); thread 0 adds the chunk sums in ascending c, starting from 0.0.
//
// wnb_mcd_dtw: one CTA per pair (grid-stride).  C(i, j) = dist(r_i, d_j) + min(C(i-1, j-1), C(i-1, j), C(i, j-1)),
// C(0, 0) = dist(r_0, d_0), row 0 and column 0 from their one predecessor; ties go to the diagonal, then (i-1, j), then
// (i, j-1).  The matrix is swept as anti-diagonals within strips of B = WNB_MCD_DTW_THREADS rows: thread t owns row
// i0 + t of the strip (its frame in registers) and at step s computes column s - t, so each step is one anti-diagonal of
// the strip.  A thread's (i-1, j) is its neighbour's value of the previous step (two ping-pong arrays in shared memory),
// its (i-1, j-1) the (i-1, j) it read one step earlier, its (i, j-1) its own previous value; the strip's last row is kept
// for the next strip in a row buffer of Td doubles (shared memory up to WNB_MCD_DTW_SMEM_COLS columns, else the
// workspace).  The decoded frames a step needs lie in two chunks of B columns, double-buffered in shared memory.  Each
// cell's step direction is one byte of the workspace, laid out step-major per strip so that every step's stores are
// contiguous.  Thread 0 then walks the directions back from (Tr-1, Td-1) and writes the path length, and the path itself
// when asked.  Since C(i, j) = C(prev) + dist(i, j) and addition commutes, C(Tr-1, Td-1) is the sum of dist along the
// path added in forward order from (0, 0); it is written as the pair's sum.
#include "common.cuh"

namespace wnb {

constexpr int kMcdAlignedThreads = 256;
constexpr int kDtwB = WNB_MCD_DTW_THREADS;

__host__ __device__ inline unsigned long long align16(unsigned long long v) { return (v + 15ull) & ~15ull; }

// workspace bytes of one DTW pair: the row buffer (only past WNB_MCD_DTW_SMEM_COLS columns), then the direction bytes
__host__ __device__ inline unsigned long long dtw_rowbuf_bytes(long long td) {
  return td > WNB_MCD_DTW_SMEM_COLS ? align16(8ull * (unsigned long long)td) : 0ull;
}
__host__ __device__ inline unsigned long long dtw_strip_bytes(long long td) {
  return (unsigned long long)kDtwB * (unsigned long long)(td + kDtwB - 1);
}
__host__ __device__ inline unsigned long long dtw_pair_bytes(long long tr, long long td) {
  const unsigned long long strips = (unsigned long long)((tr + kDtwB - 1) / kDtwB);
  return dtw_rowbuf_bytes(td) + align16(strips * dtw_strip_bytes(td));
}

__device__ __forceinline__ double warp_sum_xor_rn(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__global__ void __launch_bounds__(kMcdAlignedThreads) mcd_aligned_kernel(
    const float* __restrict__ ref, const float* __restrict__ dec, int n_cols, const long long* __restrict__ ref_off,
    const long long* __restrict__ dec_off, int n_pairs, double* __restrict__ sum, int64_t* __restrict__ count) {
  constexpr int kWarps = kMcdAlignedThreads / 32;
  __shared__ double chunk_sum[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, D = n_cols - 1;
  for (int p = blockIdx.x; p < n_pairs; p += gridDim.x) {
    const long long r0 = ref_off[p], d0 = dec_off[p];
    const long long tr = ref_off[p + 1] - r0, td = dec_off[p + 1] - d0;
    const long long n = tr < td ? tr : td;
    const long long chunks = (n + 31) / 32;
    double acc = 0.0;
    for (long long cb = 0; cb < chunks; cb += kWarps) {
      const long long c = cb + warp;
      if (c < chunks) {
        const long long t = c * 32 + lane;
        double v = 0.0;
        if (t < n) {
          const float* a = ref + (r0 + t) * n_cols;
          const float* b = dec + (d0 + t) * n_cols;
          double s = 0.0;
          for (int d = 1; d <= D; d++) {
            const double e = __dsub_rn((double)a[d], (double)b[d]);
            s = __dadd_rn(s, __dmul_rn(e, e));
          }
          v = __dsqrt_rn(s);
        }
        v = warp_sum_xor_rn(v);
        if (lane == 0) chunk_sum[warp] = v;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        const int m = chunks - cb < kWarps ? (int)(chunks - cb) : kWarps;
        for (int w = 0; w < m; w++) acc = __dadd_rn(acc, chunk_sum[w]);
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      sum[p] = acc;
      count[p] = n;
    }
  }
}

__global__ void __launch_bounds__(kDtwB, 1) mcd_dtw_kernel(
    const float* __restrict__ ref, const float* __restrict__ dec, int n_cols, const long long* __restrict__ ref_off,
    const long long* __restrict__ dec_off, int n_pairs, unsigned char* __restrict__ ws, double* __restrict__ sum,
    int64_t* __restrict__ count, int2* __restrict__ path) {
  constexpr int B = kDtwB;
  extern __shared__ double sm[];
  __shared__ unsigned long long red[B / 32];
  __shared__ long long s_len;
  const int D = n_cols - 1, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* ring = sm;                     // [2][D][B]: decoded frames of two chunks of B columns
  double* cur = ring + 2 * D * B;        // [2][B]: C of each row at the last two steps
  double* rowbuf_sm = cur + 2 * B;       // the strip's last row, when Td <= WNB_MCD_DTW_SMEM_COLS
  const long long ref_base = ref_off[0], dec_base = dec_off[0];
  for (int p = blockIdx.x; p < n_pairs; p += gridDim.x) {
    const long long r0 = ref_off[p], d0 = dec_off[p];
    const int Tr = (int)(ref_off[p + 1] - r0), Td = (int)(dec_off[p + 1] - d0);
    // this pair's workspace: the bytes of the pairs before it (the header's layout)
    unsigned long long before = 0;
    for (int q = t; q < p; q += B) before += dtw_pair_bytes(ref_off[q + 1] - ref_off[q], dec_off[q + 1] - dec_off[q]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
    if (lane == 0) red[warp] = before;
    __syncthreads();
    before = 0;
    for (int w = 0; w < B / 32; w++) before += red[w];
    unsigned char* w0 = ws + before;
    double* rowbuf = Td > WNB_MCD_DTW_SMEM_COLS ? reinterpret_cast<double*>(w0) : rowbuf_sm;
    unsigned char* dirs = w0 + dtw_rowbuf_bytes(Td);
    const long long strip_bytes = (long long)dtw_strip_bytes(Td);
    for (int i0 = 0; i0 < Tr; i0 += B) {
      const int rows = Tr - i0 < B ? Tr - i0 : B;
      const int i = i0 + t;
      double rr[WNB_MCD_MAX_DIM];
      if (t < rows) {
        const float* a = ref + (r0 + i) * n_cols + 1;
#pragma unroll
        for (int d = 0; d < WNB_MCD_MAX_DIM; d++)
          if (d < D) rr[d] = (double)a[d];
      }
      unsigned char* sd = dirs + (long long)(i0 / B) * strip_bytes;
      double up_prev = 0.0, left = 0.0;
      const int steps = Td + rows - 1;
      for (int s = 0; s < steps; s++) {
        if ((s & (B - 1)) == 0) {      // chunk s / B of the decoded frames replaces chunk s / B - 2
          const int jl = s + t;
          if (jl < Td) {
            const float* b = dec + (d0 + jl) * n_cols + 1;
            double* slot = ring + ((s / B) & 1) * D * B + t;
            for (int d = 0; d < D; d++) slot[d * B] = (double)b[d];
          }
          __syncthreads();
        }
        const int j = s - t;
        if (t < rows && j >= 0 && j < Td) {
          const double* col = ring + ((j / B) & 1) * D * B + (j & (B - 1));
          double acc = 0.0;
#pragma unroll
          for (int d = 0; d < WNB_MCD_MAX_DIM; d++) {
            if (d < D) {
              const double e = __dsub_rn(rr[d], col[d * B]);
              acc = __dadd_rn(acc, __dmul_rn(e, e));
            }
          }
          const double dist = __dsqrt_rn(acc);
          double up = 0.0;
          if (i > 0) up = t > 0 ? cur[((s - 1) & 1) * B + t - 1] : rowbuf[j];
          double c;
          unsigned char dir;
          if (i == 0 && j == 0) {
            c = dist;
            dir = 3;
          } else if (i == 0) {
            c = __dadd_rn(dist, left);
            dir = 2;
          } else if (j == 0) {
            c = __dadd_rn(dist, up);
            dir = 1;
          } else {
            double best = up_prev;
            dir = 0;
            if (up < best) { best = up; dir = 1; }
            if (left < best) { best = left; dir = 2; }
            c = __dadd_rn(dist, best);
          }
          cur[(s & 1) * B + t] = c;
          sd[(long long)s * B + t] = dir;
          if (t == rows - 1) rowbuf[j] = c;
          if (i == Tr - 1 && j == Td - 1) sum[p] = c;
          up_prev = up;
          left = c;
        }
        __syncthreads();
      }
    }
    // the path: back from (Tr-1, Td-1), written from the end of the pair's slot of Tr + Td - 1 steps
    const long long cap = (long long)Tr + Td - 1;
    int2* pp = path ? path + ((r0 - ref_base) + (d0 - dec_base) - p) : nullptr;
    if (t == 0) {
      int bi = Tr - 1, bj = Td - 1;
      long long len = 1;
      if (pp) pp[cap - 1] = make_int2(bi, bj);
      while (bi > 0 || bj > 0) {
        if (bi == 0) {
          bj--;
        } else if (bj == 0) {
          bi--;
        } else {
          const int bt = bi & (B - 1);
          const unsigned char dir = dirs[(long long)(bi / B) * strip_bytes + (long long)(bj + bt) * B + bt];
          if (dir == 0) { bi--; bj--; } else if (dir == 1) { bi--; } else { bj--; }
        }
        len++;
        if (pp) pp[cap - len] = make_int2(bi, bj);
      }
      count[p] = len;
      s_len = len;
    }
    __syncthreads();
    const long long len = s_len;
    if (pp && len < cap) {             // move it to the start of the slot; a chunk is read before any of it is written
      for (long long c0 = 0; c0 < len; c0 += B) {
        int2 v = make_int2(0, 0);
        if (c0 + t < len) v = pp[cap - len + c0 + t];
        __syncthreads();
        if (c0 + t < len) pp[c0 + t] = v;
        __syncthreads();
      }
    }
    __syncthreads();
  }
}

// the launchers' shared checks: shapes, the host copy of the offset tables, and the largest decoded length
static int check_pairs(const char* name, int n_cols, const long long* host_ref_offsets,
                       const long long* host_dec_offsets, int n_pairs) {
  WNB_REQUIRE(n_pairs > 0, "%s: need n_pairs > 0, got %d", name, n_pairs);
  WNB_REQUIRE(host_ref_offsets && host_dec_offsets, "%s: null host offsets", name);
  if (n_cols - 1 < 1 || n_cols - 1 > WNB_MCD_MAX_DIM) {
    set_error("%s: %d columns is not supported (1 <= D <= %d, c0 and D coefficients per frame)", name, n_cols,
              WNB_MCD_MAX_DIM);
    return WNB_ERR_UNSUPPORTED;
  }
  WNB_REQUIRE(host_ref_offsets[0] >= 0 && host_dec_offsets[0] >= 0, "%s: negative frame offset", name);
  for (int p = 0; p < n_pairs; p++) {
    const long long tr = host_ref_offsets[p + 1] - host_ref_offsets[p];
    const long long td = host_dec_offsets[p + 1] - host_dec_offsets[p];
    if (tr < 1 || td < 1 || tr > WNB_MCD_MAX_FRAMES || td > WNB_MCD_MAX_FRAMES) {
      set_error("%s: pair %d has %lld reference and %lld decoded frames (each side needs 1 to %d)", name, p, tr, td,
                WNB_MCD_MAX_FRAMES);
      return WNB_ERR_UNSUPPORTED;
    }
  }
  return WNB_OK;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_mcd_aligned(const float* ref, const float* dec, int n_cols, const long long* ref_offsets,
                            const long long* dec_offsets, const long long* host_ref_offsets,
                            const long long* host_dec_offsets, int n_pairs, double* sum, int64_t* count,
                            void* stream) {
  const int rc = check_pairs("mcd_aligned", n_cols, host_ref_offsets, host_dec_offsets, n_pairs);
  if (rc != WNB_OK) return rc;
  WNB_REQUIRE(ref && dec && ref_offsets && dec_offsets && sum && count, "mcd_aligned: null pointer");
  const int grid = n_pairs < 65535 ? n_pairs : 65535;
  mcd_aligned_kernel<<<grid, kMcdAlignedThreads, 0, (cudaStream_t)stream>>>(ref, dec, n_cols, ref_offsets, dec_offsets,
                                                                             n_pairs, sum, count);
  WNB_CHECK_LAUNCH("mcd_aligned");
  return WNB_OK;
}

WNB_API size_t wnb_mcd_dtw_workspace(long long ref_frames, long long dec_frames) {
  if (ref_frames < 1 || dec_frames < 1 || ref_frames > WNB_MCD_MAX_FRAMES || dec_frames > WNB_MCD_MAX_FRAMES) return 0;
  return (size_t)dtw_pair_bytes(ref_frames, dec_frames);
}

WNB_API int wnb_mcd_dtw(const float* ref, const float* dec, int n_cols, const long long* ref_offsets,
                        const long long* dec_offsets, const long long* host_ref_offsets,
                        const long long* host_dec_offsets, int n_pairs, void* workspace, size_t workspace_bytes,
                        double* sum, int64_t* count, int32_t* path, void* stream) {
  const int rc = check_pairs("mcd_dtw", n_cols, host_ref_offsets, host_dec_offsets, n_pairs);
  if (rc != WNB_OK) return rc;
  WNB_REQUIRE(ref && dec && ref_offsets && dec_offsets && sum && count && workspace, "mcd_dtw: null pointer");
  WNB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "mcd_dtw: workspace is not 16-byte aligned");
  WNB_REQUIRE((reinterpret_cast<uintptr_t>(path) & 7) == 0, "mcd_dtw: path is not 8-byte aligned");
  unsigned long long need = 0;
  long long row_cols = 0;
  for (int p = 0; p < n_pairs; p++) {
    const long long td = host_dec_offsets[p + 1] - host_dec_offsets[p];
    need += dtw_pair_bytes(host_ref_offsets[p + 1] - host_ref_offsets[p], td);
    if (td <= WNB_MCD_DTW_SMEM_COLS && td > row_cols) row_cols = td;
  }
  WNB_REQUIRE(need <= workspace_bytes, "mcd_dtw: the pairs need %llu workspace bytes, %zu given", need,
              workspace_bytes);
  const int D = n_cols - 1;
  const size_t smem = sizeof(double) * (2 * (size_t)D * kDtwB + 2 * kDtwB + (size_t)row_cols);
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(mcd_dtw_kernel), smem));
  int per_sm = 0;
  WNB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mcd_dtw_kernel, kDtwB, smem));
  const long long slots = (long long)device_sms() * (per_sm > 0 ? per_sm : 1);
  const int grid = (int)(n_pairs < slots ? n_pairs : slots);
  mcd_dtw_kernel<<<grid, kDtwB, smem, (cudaStream_t)stream>>>(ref, dec, n_cols, ref_offsets, dec_offsets, n_pairs,
                                                              static_cast<unsigned char*>(workspace), sum, count,
                                                              reinterpret_cast<int2*>(path));
  WNB_CHECK_LAUNCH("mcd_dtw");
  return WNB_OK;
}

}  // extern "C"
