// stockham.cuh -- the in-shared-memory radix-2 Stockham FFT shared by the feature kernels (melspc.cu, mcep.cu).
#pragma once

namespace wnb {

// Forward FFT (exp(-2 pi i n k / N)) of length N = 2^log2n by the whole block.  re / im hold the input (separate real and
// imaginary arrays); re2 / im2 are scratch of the same size.  The pointers are swapped each stage (ping-pong), so on
// return re / im point at the natural-order output and re2 / im2 at the scratch.  twiddles: N / 2 interleaved pairs
// (cos, -sin)(2 pi m / N) in global memory.  Stage s (Ns = 2^s) combines pairs j, j + N/2 with twiddle
// exp(-2 pi i k / (2 Ns)), k = j mod Ns, = twiddles[k * N / (2 Ns)], and writes positions (j - k) * 2 + k and that + Ns.
// The caller must __syncthreads() after writing the input; the function ends with one.
__device__ __forceinline__ void stockham_fft(double*& re, double*& im, double*& re2, double*& im2, int N, int log2n,
                                             const double* __restrict__ twiddles) {
  const int half = N >> 1;
  for (int s = 0; s < log2n; s++) {
    const int Ns = 1 << s;
    for (int j = threadIdx.x; j < half; j += blockDim.x) {
      const int k = j & (Ns - 1);
      const int m = k << (log2n - 1 - s);
      const double wr = twiddles[2 * m], wi = twiddles[2 * m + 1];
      const double ar = re[j], ai = im[j], br = re[j + half], bi = im[j + half];
      const double tr = fma(br, wr, -(bi * wi));
      const double ti = fma(br, wi, bi * wr);
      const int o = ((j - k) << 1) + k;
      re2[o] = ar + tr;
      im2[o] = ai + ti;
      re2[o + Ns] = ar - tr;
      im2[o + Ns] = ai - ti;
    }
    __syncthreads();
    double* t = re; re = re2; re2 = t;
    t = im; im = im2; im2 = t;
  }
}

}  // namespace wnb
