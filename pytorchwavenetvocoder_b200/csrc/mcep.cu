// mcep.cu -- wnb_mcep: the reference's STFT mel-cepstra (bin/feature_extract.py --feature_type mcep: stft_mcep, one
// pysptk.mcep(frame, order, alpha, eps=1e-10, etype=1) per frame) for a BATCH of utterances on the GPU, float64
// throughout and one float32 rounding at the end.
//
// One block per frame.  Frame t of an utterance is x[t hop, t hop + fftl) in int16 units (no padding, no centring),
// times the periodic Hamming window; a radix-2 Stockham FFT in shared memory (stockham.cuh, the one melspc.cu uses)
// gives the periodogram P_k = |X_k|^2 + eps, k = 0 .. fftl / 2.  Mel-cepstral analysis minimises
// E(c) = sum_k [P_k / |H_k|^2 - log(P_k / |H_k|^2) - 1] with log|H_k| = sum_m c_m cos(m w~_k) on the alpha-warped axis
// by Newton-Raphson, as SPTK's mcep does, but every frequency warp is evaluated as a sum over the bins instead of SPTK's
// FFTs and truncated freqt / frqtr recursions:
//   - initial value: c = W log P (W: the host's (order + 2) x (fftl / 2 + 1) table of the linear map "real cepstrum of
//     log P, halve c[0] and c[L/2], freqt to the order"; its last row gives the halved c[0] that seeds the convergence
//     test), one warp per row, lanes over bins, xor-butterfly sum;
//   - each iteration: log|H_k| by Clenshaw from cos w~_k (host table), R_k = P_k / exp(2 log|H_k|) times the bin's
//     multiplicity (1 at k = 0 and fftl / 2, else 2), r(i) = (1/fftl) sum_k R_k T_i(cos w~_k) for i = 0 .. 2 order with
//     the Chebyshev recurrence per bin (MC_CHUNK values of i per pass, the recurrence state kept per bin in shared
//     memory), per-thread sums in ascending k, xor-butterfly warp sums, warps summed in order;
//   - the convergence test (from iteration miniter: |(r0 - s) / r0| < threshold stops BEFORE the update, else s = r0);
//   - the update d solves (T + H) d = r(0 .. order) - (-alpha)^(0 .. order), T_ij = r(|i - j|), H_ij = r(i + j), by an
//     LL^T Cholesky factorisation in shared memory by one warp; a pivot below min_det fails the frame.
// iters[frame] = updates applied (j - 1 when the test at iteration j converges, else maxiter), -j when the solve of
// iteration j fails.  The bin sums equal SPTK's recursions up to the recursions' truncation at fftl / 2 terms, which is
// below 1e-13 inside the supported range (include/wnb200.h).  No atomics, fixed orders: two runs are bit-identical.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wnb200.h"
#include "common.cuh"
#include "stockham.cuh"

namespace wnb {

constexpr int MC_THREADS_MAX = 256;
constexpr int MC_CHUNK = 8;       // r(i) values accumulated per pass over the bins

// sum over the warp by an xor butterfly: every lane ends with the same, order-fixed value
__device__ __forceinline__ double warp_sum_xor(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(MC_THREADS_MAX) mcep_kernel(
    const void* __restrict__ xin, int x_i16, const long long* __restrict__ offsets,
    const long long* __restrict__ frame_offsets, int n_utts, int fftl, int log2n, int hop, int order,
    const double* __restrict__ window, const double* __restrict__ twiddles, const double* __restrict__ warp_cos,
    const double* __restrict__ init_map, const double* __restrict__ neg_alpha_pow, int miniter, int maxiter,
    double threshold, double eps, double min_det, float* __restrict__ out, int32_t* __restrict__ iters) {
  extern __shared__ double sm[];
  const int N = fftl, nb = (N >> 1) + 1, n = order + 1, J = 2 * order + 1;
  const int nw = blockDim.x >> 5, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double* re = sm;
  double* im = sm + N;
  double* re2 = sm + 2 * N;
  double* im2 = sm + 3 * N;
  double* A = sm + 4 * N;                 // n x n: T + H, then its Cholesky factor (lower triangle)
  double* r = A + n * n;                  // r(0 .. 2 order)
  double* part = r + J;                   // per-warp partial sums, nw x MC_CHUNK
  double* mc = part + nw * MC_CHUNK;      // the mel-cepstrum being iterated
  double* vec = mc + n;                   // right-hand side, then the update
  double* misc = vec + n;                 // [0] convergence seed s, [1] converged (1) or not (0), [2] the solve failed
  const long long f = blockIdx.x;
  // the utterance of frame f: the last u with frame_offsets[u] <= f
  int lo = 0, hi = n_utts;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (frame_offsets[mid] <= f) lo = mid; else hi = mid;
  }
  const long long j0 = offsets[lo] + (f - frame_offsets[lo]) * hop;
  const int16_t* x16 = reinterpret_cast<const int16_t*>(xin);
  const double* x64 = reinterpret_cast<const double*>(xin);
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    re[i] = (x_i16 ? (double)x16[j0 + i] : x64[j0 + i]) * window[i];
    im[i] = 0.0;
  }
  __syncthreads();
  stockham_fft(re, im, re2, im2, N, log2n, twiddles);
  // re / im: X; re2 .. re2 + 2N: free (im2 == re2 + N whichever way the ping-pong ended)
  double* P = re2;
  double* cw = re2 + nb;
  double* R = re2 + 2 * nb;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    P[k] = __dadd_rn(__dadd_rn(__dmul_rn(re[k], re[k]), __dmul_rn(im[k], im[k])), eps);
    cw[k] = warp_cos[k];
  }
  __syncthreads();
  double* Ta = re;                        // per bin: T_i(cos w~_k) at the start of the next pass over the bins
  double* Tb = re + nb;                   // and T_{i+1}
  for (int k = threadIdx.x; k < nb; k += blockDim.x) R[k] = log(P[k]);
  __syncthreads();
  for (int row = wid; row <= n; row += nw) {
    const double* w = init_map + (size_t)row * nb;
    double acc = 0.0;
    for (int k = lane; k < nb; k += 32) acc = fma(w[k], R[k], acc);
    acc = warp_sum_xor(acc);
    if (lane == 0) {
      if (row < n) mc[row] = acc; else misc[0] = acc;
    }
  }
  __syncthreads();
  const double inv_n = 1.0 / (double)N;   // a power of two: exact
  int count = maxiter;
  for (int j = 1; j <= maxiter; j++) {
    for (int k = threadIdx.x; k < nb; k += blockDim.x) {
      const double x = cw[k], x2 = x + x;
      double b1 = 0.0, b2 = 0.0;
      for (int m = order; m >= 1; m--) {
        const double b0 = fma(x2, b1, mc[m] - b2);
        b2 = b1;
        b1 = b0;
      }
      const double lh = fma(x, b1, mc[0] - b2);
      const double v = P[k] / exp(lh + lh);
      R[k] = (k == 0 || k == nb - 1) ? v : v + v;
      Ta[k] = 1.0;
      Tb[k] = x;
    }
    __syncthreads();
    for (int i0 = 0; i0 < J; i0 += MC_CHUNK) {
      double acc[MC_CHUNK];
#pragma unroll
      for (int c = 0; c < MC_CHUNK; c++) acc[c] = 0.0;
      for (int k = threadIdx.x; k < nb; k += blockDim.x) {
        const double x2 = cw[k] + cw[k], Rk = R[k];
        double a = Ta[k], b = Tb[k];
#pragma unroll
        for (int c = 0; c < MC_CHUNK; c++) {
          acc[c] = fma(Rk, a, acc[c]);
          const double t = fma(x2, b, -a);
          a = b;
          b = t;
        }
        Ta[k] = a;
        Tb[k] = b;
      }
#pragma unroll
      for (int c = 0; c < MC_CHUNK; c++) acc[c] = warp_sum_xor(acc[c]);
      if (lane == 0) {
#pragma unroll
        for (int c = 0; c < MC_CHUNK; c++) part[wid * MC_CHUNK + c] = acc[c];
      }
      __syncthreads();
      if (threadIdx.x < MC_CHUNK && i0 + (int)threadIdx.x < J) {
        double v = 0.0;
        for (int w = 0; w < nw; w++) v += part[w * MC_CHUNK + threadIdx.x];
        r[i0 + threadIdx.x] = v * inv_n;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      int state = 0;
      if (j >= miniter) {
        const double t = r[0];
        if (fabs((t - misc[0]) / t) < threshold) state = 1; else misc[0] = t;
      }
      misc[1] = (double)state;
    }
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
      const int i = e / n, k = e - i * n;
      A[e] = r[i > k ? i - k : k - i] + r[i + k];
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) vec[i] = r[i] - neg_alpha_pow[i];
    __syncthreads();
    if (misc[1] == 1.0) {
      count = j - 1;
      break;
    }
    if (wid == 0) {
      bool bad = false;
      for (int c = 0; c < n; c++) {           // column c of L, left-looking, sums in ascending k
        for (int i = c + lane; i < n; i += 32) {
          double v = A[i * n + c];
          for (int k = 0; k < c; k++) v = fma(-A[i * n + k], A[c * n + k], v);
          A[i * n + c] = v;
        }
        __syncwarp();
        const double s = A[c * n + c];
        if (!(s >= min_det)) { bad = true; break; }
        const double l = sqrt(s);
        __syncwarp();
        for (int i = c + lane; i < n; i += 32) A[i * n + c] = i == c ? l : A[i * n + c] / l;
        __syncwarp();
      }
      if (!bad) {
        for (int c = 0; c < n; c++) {         // L y = b
          const double y = vec[c] / A[c * n + c];
          __syncwarp();
          if (lane == 0) vec[c] = y;
          for (int i = c + 1 + lane; i < n; i += 32) vec[i] = fma(-A[i * n + c], y, vec[i]);
          __syncwarp();
        }
        for (int c = n - 1; c >= 0; c--) {    // L^T d = y
          const double d = vec[c] / A[c * n + c];
          __syncwarp();
          if (lane == 0) vec[c] = d;
          for (int i = lane; i < c; i += 32) vec[i] = fma(-A[c * n + i], d, vec[i]);
          __syncwarp();
        }
      }
      if (lane == 0) misc[2] = bad ? 1.0 : 0.0;
    }
    __syncthreads();
    if (misc[2] == 1.0) {
      count = -j;
      break;
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) mc[i] += vec[i];
    __syncthreads();
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) out[(size_t)f * n + i] = __double2float_rn(mc[i]);
  if (threadIdx.x == 0) iters[f] = count;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_mcep(const void* x, int x_is_i16, const long long* offsets, const long long* frame_offsets, int n_utts,
                     long long n_frames, int fftl, int hop, int order, double alpha, const double* window,
                     const double* twiddles, const double* warp_cos, const double* init_map,
                     const double* neg_alpha_pow, int miniter, int maxiter, double threshold, double eps,
                     double min_det, float* out, int32_t* iters, void* stream) {
  WNB_REQUIRE(x && offsets && frame_offsets && window && twiddles && warp_cos && init_map && neg_alpha_pow && out && iters,
              "mcep: null pointer");
  WNB_REQUIRE(n_utts > 0 && n_frames >= n_utts && n_frames <= 0x7fffffffLL,
              "mcep: need n_utts > 0 and n_utts <= n_frames < 2^31 (n_utts %d, n_frames %lld)", n_utts, n_frames);
  WNB_REQUIRE(hop > 0, "mcep: need hop > 0, got %d", hop);
  WNB_REQUIRE(maxiter >= 0 && maxiter <= WNB_MCEP_MAX_ITER && miniter >= 0,
              "mcep: need 0 <= maxiter <= %d and miniter >= 0 (miniter %d, maxiter %d)", WNB_MCEP_MAX_ITER, miniter,
              maxiter);
  WNB_REQUIRE(eps > 0.0 && eps < 1e300 && threshold >= 0.0 && min_det >= 0.0,
              "mcep: need eps > 0, threshold >= 0 and min_det >= 0");
  int log2n = 0;
  while ((1 << log2n) < fftl && log2n < 30) log2n++;
  if (fftl < WNB_MCEP_MIN_FFTL || fftl > WNB_MCEP_MAX_FFTL || (1 << log2n) != fftl || order < 1 ||
      order > WNB_MCEP_MAX_ORDER || !(alpha >= 0.0 && alpha <= WNB_MCEP_MAX_ALPHA)) {
    set_error("mcep: fftl %d, order %d, alpha %g is not supported (fftl a power of two from %d to %d, 1 <= order <= %d, "
              "0 <= alpha <= %g)", fftl, order, alpha, WNB_MCEP_MIN_FFTL, WNB_MCEP_MAX_FFTL, WNB_MCEP_MAX_ORDER,
              WNB_MCEP_MAX_ALPHA);
    return WNB_ERR_UNSUPPORTED;
  }
  const int threads = fftl / 2 < MC_THREADS_MAX ? fftl / 2 : MC_THREADS_MAX;
  const int n = order + 1;
  const size_t smem = sizeof(double) * (4 * (size_t)fftl + (size_t)n * n + (2 * order + 1) +
                                        (size_t)(threads / 32) * MC_CHUNK + 2 * n + 3);
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(mcep_kernel), smem));
  mcep_kernel<<<(unsigned)n_frames, threads, smem, (cudaStream_t)stream>>>(
      x, x_is_i16, offsets, frame_offsets, n_utts, fftl, log2n, hop, order, window, twiddles, warp_cos, init_map,
      neg_alpha_pow, miniter, maxiter, threshold, eps, min_det, out, iters);
  WNB_CHECK_LAUNCH("mcep");
  return WNB_OK;
}

}  // extern "C"
