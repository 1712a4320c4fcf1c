// melspc.cu -- wnb_melspc_lowcut / wnb_melspc: the reference's mel-spectrogram features (bin/feature_extract.py
// --feature_type melspc: low_cut_filter, librosa.feature.melspectrogram(power=1), log10(max(1e-10, .))) for a BATCH of
// utterances on the GPU, float64 throughout and one float32 rounding at the end.
//
// Low-cut FIR (lowcut_kernel): y[n] = sum_k b[k] x[n - k] with x[< 0] = 0 (scipy lfilter(b, 1, x): zero initial state,
// output as long as the input).  One block computes LC_TILE consecutive outputs of one utterance from a shared-memory copy
// of the samples [tile - (n_taps - 1), tile + LC_TILE); each output is one fma chain in ascending k.  Optionally the int16
// wav the reference writes (np.int16 of the float64 result: C truncation to int32, low 16 bits kept).
//
// Frames (melspc_kernel): one block per frame.  Frame t of an utterance of length n reads padded positions
// [t hop, t hop + fftl) of np.pad(x / 32768, fftl / 2, mode="reflect") through a closed-form index map, multiplies by the
// window, runs a radix-2 Stockham FFT of length fftl in shared memory (stockham.cuh: separate re / im arrays, ping-pong,
// natural-order output, host float64 twiddles), takes |X[k]| with hypot for k = 0 .. fftl / 2, and sums each mel
// filter's nonzero bins [lo, hi) in ascending order against the float32 filterbank widened to float64.  Then log10(max(1e-10, .)) in float64
// and one float32 rounding; the row goes to out[frame_offsets[u] + t][m].  No atomics: two runs are bit-identical.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wnb200.h"
#include "common.cuh"
#include "melspc_frame.cuh"

namespace wnb {

constexpr int LC_TILE = 1024;     // outputs per low-cut block
constexpr int LC_THREADS = 256;
constexpr int MS_THREADS_MAX = 256;

// np.int16(v) of a float64 on x86-64: cvttsd2si to int32 (out of range and NaN give INT_MIN), then the low 16 bits.
__device__ __forceinline__ int16_t np_int16(double v) {
  const int32_t i = (v > -2147483649.0 && v < 2147483648.0) ? (int32_t)v : (int32_t)0x80000000u;
  return (int16_t)i;
}

__global__ void __launch_bounds__(LC_THREADS) lowcut_kernel(const void* __restrict__ xin, int x_i16,
                                                            const long long* __restrict__ offsets,
                                                            const double* __restrict__ taps, int n_taps,
                                                            double* __restrict__ y, int16_t* __restrict__ y16) {
  extern __shared__ double sm[];
  double* b = sm;                         // taps[0 .. n_taps)
  double* xs = sm + n_taps;               // x[tile0 - (n_taps - 1) + i], i < LC_TILE + n_taps - 1
  const int u = blockIdx.y;
  const long long off = offsets[u], len = offsets[u + 1] - off;
  const long long tile0 = (long long)blockIdx.x * LC_TILE;
  if (tile0 >= len) return;
  const int16_t* x16 = reinterpret_cast<const int16_t*>(xin);
  const double* x64 = reinterpret_cast<const double*>(xin);
  for (int i = threadIdx.x; i < n_taps; i += LC_THREADS) b[i] = taps[i];
  const int span = LC_TILE + n_taps - 1;
  for (int i = threadIdx.x; i < span; i += LC_THREADS) {
    const long long n = tile0 - (n_taps - 1) + i;
    xs[i] = (n >= 0 && n < len) ? (x_i16 ? (double)x16[off + n] : x64[off + n]) : 0.0;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < LC_TILE; r += LC_THREADS) {
    const long long n = tile0 + r;
    if (n >= len) break;
    const double acc = lowcut_fma(b, n_taps, xs + r + (n_taps - 1));   // xr[-k] = x[n - k]
    y[off + n] = acc;
    if (y16 != nullptr) y16[off + n] = np_int16(acc);
  }
}

__global__ void __launch_bounds__(MS_THREADS_MAX) melspc_kernel(
    const void* __restrict__ xin, int x_i16, const long long* __restrict__ offsets,
    const long long* __restrict__ frame_offsets, int n_utts, int fftl, int log2n, int hop,
    const double* __restrict__ window, const double* __restrict__ twiddles, const float* __restrict__ mel_basis,
    const int32_t* __restrict__ mel_lo, const int32_t* __restrict__ mel_hi, int n_mels, float* __restrict__ out) {
  extern __shared__ double sm[];
  const int N = fftl, half = fftl >> 1, nb = half + 1;
  double* re = sm;
  double* im = sm + N;
  double* re2 = sm + 2 * N;
  double* im2 = sm + 3 * N;
  const long long f = blockIdx.x;
  // the utterance of frame f: the last u with frame_offsets[u] <= f
  int lo = 0, hi = n_utts;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (frame_offsets[mid] <= f) lo = mid; else hi = mid;
  }
  const long long off = offsets[lo], len = offsets[lo + 1] - off;
  const long long start = (f - frame_offsets[lo]) * hop - half;   // signal index of the frame's first sample
  const int16_t* x16 = reinterpret_cast<const int16_t*>(xin);
  const double* x64 = reinterpret_cast<const double*>(xin);
  melspc_frame(
      [&](int n) {
        const long long j = off + reflect_index(start + n, len);
        return x_i16 ? (double)x16[j] : x64[j];
      },
      [&](int m, float v) { out[(size_t)f * n_mels + m] = v; }, re, im, re2, im2, N, nb, log2n, window, twiddles,
      mel_basis, mel_lo, mel_hi, n_mels);
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_melspc_lowcut(const void* x, int x_is_i16, const long long* offsets, int n_utts, long long max_len,
                              const double* taps, int n_taps, double* y, int16_t* y16, void* stream) {
  WNB_REQUIRE(x && offsets && taps && y, "melspc_lowcut: null pointer");
  WNB_REQUIRE(n_utts > 0 && n_utts <= 65535, "melspc_lowcut: need 0 < n_utts <= 65535, got %d", n_utts);
  WNB_REQUIRE(max_len > 0 && max_len <= (long long)LC_TILE * 0x7fffffffLL, "melspc_lowcut: bad max_len %lld", max_len);
  WNB_REQUIRE(n_taps >= 1 && n_taps <= WNB_MELSPC_MAX_TAPS, "melspc_lowcut: need 1 <= n_taps <= %d, got %d",
              WNB_MELSPC_MAX_TAPS, n_taps);
  const size_t smem = sizeof(double) * ((size_t)n_taps + LC_TILE + n_taps - 1);
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(lowcut_kernel), smem));
  const dim3 grid((unsigned)((max_len + LC_TILE - 1) / LC_TILE), (unsigned)n_utts);
  lowcut_kernel<<<grid, LC_THREADS, smem, (cudaStream_t)stream>>>(x, x_is_i16, offsets, taps, n_taps, y, y16);
  WNB_CHECK_LAUNCH("melspc_lowcut");
  return WNB_OK;
}

WNB_API int wnb_melspc(const void* x, int x_is_i16, const long long* offsets, const long long* frame_offsets, int n_utts,
                       long long n_frames, int fftl, int hop, const double* window, const double* twiddles,
                       const float* mel_basis, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, float* out,
                       void* stream) {
  WNB_REQUIRE(x && offsets && frame_offsets && window && twiddles && mel_basis && mel_lo && mel_hi && out,
              "melspc: null pointer");
  WNB_REQUIRE(n_utts > 0 && n_frames >= n_utts && n_frames <= 0x7fffffffLL,
              "melspc: need n_utts > 0 and n_utts <= n_frames < 2^31 (n_utts %d, n_frames %lld)", n_utts, n_frames);
  WNB_REQUIRE(hop > 0 && n_mels > 0, "melspc: need hop > 0 and n_mels > 0 (hop %d, n_mels %d)", hop, n_mels);
  int log2n = 0;
  while ((1 << log2n) < fftl && log2n < 30) log2n++;
  if (fftl < WNB_MELSPC_MIN_FFTL || fftl > WNB_MELSPC_MAX_FFTL || (1 << log2n) != fftl) {
    set_error("melspc: fftl %d is not supported (powers of two from %d to %d)", fftl, WNB_MELSPC_MIN_FFTL,
              WNB_MELSPC_MAX_FFTL);
    return WNB_ERR_UNSUPPORTED;
  }
  const size_t smem = sizeof(double) * 4 * (size_t)fftl;
  const int threads = fftl / 2 < MS_THREADS_MAX ? fftl / 2 : MS_THREADS_MAX;
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(melspc_kernel), smem));
  melspc_kernel<<<(unsigned)n_frames, threads, smem, (cudaStream_t)stream>>>(
      x, x_is_i16, offsets, frame_offsets, n_utts, fftl, log2n, hop, window, twiddles, mel_basis, mel_lo, mel_hi, n_mels,
      out);
  WNB_CHECK_LAUNCH("melspc");
  return WNB_OK;
}

}  // extern "C"
