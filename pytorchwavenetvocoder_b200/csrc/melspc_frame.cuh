// melspc_frame.cuh -- the per-sample FIR step and the per-frame body shared by the whole-file melspc kernels
// (melspc.cu) and the streaming ones (melspc_stream.cu), so that both compute every feature with the same instructions
// in the same order: a streamed frame is bit-identical to the same frame of the whole file.
#pragma once
#include <stdint.h>

#include "stockham.cuh"

namespace wnb {

// One low-cut output y[n] = sum_{k < n_taps} b[k] x[n - k], one fma chain in ascending k, with xr[-k] = x[n - k].
__device__ __forceinline__ double lowcut_fma(const double* b, int n_taps, const double* xr) {
  double acc = 0.0;
#pragma unroll 5
  for (int k = 0; k < n_taps; k++) acc = fma(b[k], xr[-k], acc);
  return acc;
}

// np.pad(x, pad, mode="reflect") index map for a signal of length n >= 1 and a position i in [-pad, n + pad): numpy's
// reflection (edge sample not repeated) is periodic with period 2 (n - 1); a one-sample signal repeats its sample.
__device__ __forceinline__ long long reflect_index(long long i, long long n) {
  if (n == 1) return 0;
  const long long p = 2 * (n - 1);
  long long j = i % p;
  if (j < 0) j += p;
  return j < n ? j : p - j;
}

// One frame by the whole block.  load(n) gives the frame's n-th sample in int16 units (n < fftl, reflect padding
// already applied); store(m, v) receives the float32 feature of mel filter m.  re, im, re2, im2: fftl doubles of shared
// memory each; nb = fftl / 2 + 1.
// Window, Stockham FFT, S[k] = hypot(Re, Im) for k <= fftl / 2, each mel filter's nonzero bins in ascending order against
// the float32 table widened to float64, log10(max(1e-10, .)) and one float32 rounding.
template <class Load, class Store>
__device__ __forceinline__ void melspc_frame(const Load& load, const Store& store, double*& re, double*& im,
                                             double*& re2, double*& im2, int N, int nb, int log2n,
                                             const double* __restrict__ window, const double* __restrict__ twiddles,
                                             const float* __restrict__ mel_basis, const int32_t* __restrict__ mel_lo,
                                             const int32_t* __restrict__ mel_hi, int n_mels) {
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const double v = load(n) * 0x1p-15;   // x / 32768: exact
    re[n] = v * window[n];
    im[n] = 0.0;
  }
  __syncthreads();
  stockham_fft(re, im, re2, im2, N, log2n, twiddles);
  double* S = re2;                        // |X[k]|, k = 0 .. N/2
  for (int k = threadIdx.x; k < nb; k += blockDim.x) S[k] = hypot(re[k], im[k]);
  __syncthreads();
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    const float* w = mel_basis + (size_t)m * nb;
    double acc = 0.0;
    for (int k = mel_lo[m]; k < mel_hi[m]; k++) acc = fma((double)w[k], S[k], acc);
    store(m, __double2float_rn(log10(fmax(1e-10, acc))));
  }
}

}  // namespace wnb
