// loader.cu -- the arithmetic of the reference's train_generator (bin/train.py:67-312) on the device.
//
// The reference prepares every mini-batch on the host: slice a window out of the concatenated utterances, mu-law
// encode the WHOLE window (receptive field included, so every sample is encoded ~1.15 times), StandardScaler the
// features, transpose, stack, and copy three tensors to the GPU (train.py:157-185).  Here the concatenated waveform
// (float32) and frame-rate features stay resident in device ring buffers (uploaded once per utterance, asynchronously,
// from pinned memory) and ONE kernel cuts a whole batch out of them:
//   s0_b = s0 + b * hop                                                       (windows hop by batch_length, :178, :226)
//   x[b][i] = encode_mu_law(wave[s0_b + i])          t[b][i] = encode_mu_law(wave[s0_b + i + 1])      (train.py:167-169)
//   h[b][d][j] = float32((feat[row][d] - mean[d]) / scale[d])     row = s0_b / U + j   (up-sampling layer, :202-224)
//                                                                  row = frame_of_sample[s0_b + j]   (extend_time, :172-176)
// Positions are absolute stream positions; the buffers are rings (index = position mod capacity).
// in the dtypes numpy / sklearn use (see mulaw_encode_f32_kernel in elementwise.cu; StandardScaler.transform on a
// float32 array rounds to float32 after the subtraction and after the division -- in float64 arithmetic with
// scikit-learn 0.22, in float32 arithmetic with scikit-learn >= 1.x, selectable -- on float64 once at the final .float()).
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/wnb200.h"
#include "common.cuh"

namespace wnb {

__device__ __forceinline__ int64_t mulaw_f32(float v, float mu, double log1pmu) {
  const float sgn = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
  const float arg = __fadd_rn(1.0f, __fmul_rn(mu, fabsf(v)));
  const float lg = (float)log((double)arg);
  const float num = __fmul_rn(sgn, lg);
  const double fx = __ddiv_rn((double)num, log1pmu);
  const double q = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(fx, 1.0), 2.0), (double)mu), 0.5);
  return (int64_t)floor(q);
}

// StandardScaler.transform of one stored feature value (feat_f64: 1 = float64 rows; 0 / 2 = float32 rows, the
// scikit-learn 0.22 / >= 1.x arithmetic of device_loader._f32_scaler_mode), or the value itself when mean is NULL
__device__ __forceinline__ float scaled_feat(const void* __restrict__ feat, int64_t idx, int d,
                                            const double* __restrict__ mean, const double* __restrict__ scale,
                                            int feat_f64) {
  if (feat_f64 == 1) {
    const double v = reinterpret_cast<const double*>(feat)[idx];
    return mean ? (float)__ddiv_rn(__dadd_rn(v, -mean[d]), scale[d]) : (float)v;
  }
  const float v = reinterpret_cast<const float*>(feat)[idx];
  if (mean && feat_f64 == 2) {
    // scikit-learn >= 1.x: X -= astype(mean_, float32); X /= astype(scale_, float32)  (float32 arithmetic)
    return __fdiv_rn(__fsub_rn(v, (float)mean[d]), (float)scale[d]);
  }
  if (mean) {
    // scikit-learn 0.22 (the reference's pin): in-place ops with float64 operands, rounded to float32 after each
    const float c = (float)__dadd_rn((double)v, -mean[d]);   // X -= mean_
    return (float)__ddiv_rn((double)c, scale[d]);             // X /= scale_
  }
  return v;
}

__global__ void __launch_bounds__(256) make_train_batch_kernel(
    const float* __restrict__ wave, const void* __restrict__ feat, const int32_t* __restrict__ frame_of_sample,
    int64_t s0, int64_t hop, int U, int64_t cap_s, int64_t cap_f, const double* __restrict__ mean,
    const double* __restrict__ scale, int64_t* __restrict__ x, int64_t* __restrict__ t, float* __restrict__ h, int B, int T,
    int Tf, int D, int feat_f64, float mu, double log1pmu) {
  const int b = blockIdx.y;
  const int64_t so = s0 + (int64_t)b * hop;
  // ---- waveform: x and the next-sample targets (each sample encoded once, written to both) ----
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= T; i += gridDim.x * blockDim.x) {
    const int64_t q = mulaw_f32(__ldg(wave + (so + i) % cap_s), mu, log1pmu);
    if (i < T) x[(int64_t)b * T + i] = q;
    if (i > 0) t[(int64_t)b * T + i - 1] = q;
  }
  // ---- aux features: (frames, D) rows -> (D, Tf) with the scaler applied ----
  const int64_t fo = so / U;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < D * Tf; e += gridDim.x * blockDim.x) {
    const int d = e / Tf, j = e - d * Tf;
    const int64_t row = (frame_of_sample ? (int64_t)frame_of_sample[(so + j) % cap_s] : fo + j) % cap_f;
    h[((int64_t)b * D + d) * Tf + j] = scaled_feat(feat, row * D + d, d, mean, scale, feat_f64);
  }
}

// Corpus index of stream position p: the utterance k with starts[k] <= p < starts[k + 1] (binary search over the
// epoch table: stream start and corpus offset of every non-empty utterance, starts strictly increasing), then its offset.
__device__ __forceinline__ int64_t corpus_index(const int64_t* __restrict__ starts, const int64_t* __restrict__ offsets,
                                                int n, int64_t p) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(starts + mid) <= p) lo = mid; else hi = mid - 1;
  }
  return __ldg(offsets + lo) + (p - __ldg(starts + lo));
}

// make_train_batch_kernel's windows cut from a device-resident corpus instead of rings: the stream of concatenated
// utterances in epoch order is the table (starts, offsets); the waveform is int16 (x / 32768 is exact in float32, the
// value soundfile's float32 read gives); feature rows are those of the frame's first sample, (offset) / U.
__global__ void __launch_bounds__(256) make_train_batch_corpus_kernel(
    const int16_t* __restrict__ wave, const void* __restrict__ feat, const int64_t* __restrict__ starts,
    const int64_t* __restrict__ offsets, int n_utts, int64_t s0, int64_t hop, int U, const double* __restrict__ mean,
    const double* __restrict__ scale, int64_t* __restrict__ x, int64_t* __restrict__ t, float* __restrict__ h, int B, int T,
    int Tf, int D, int feat_f64, float mu, double log1pmu) {
  const int b = blockIdx.y;
  const int64_t so = s0 + (int64_t)b * hop;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= T; i += gridDim.x * blockDim.x) {
    const float v = __fmul_rn((float)__ldg(wave + corpus_index(starts, offsets, n_utts, so + i)), 1.0f / 32768.0f);
    const int64_t q = mulaw_f32(v, mu, log1pmu);
    if (i < T) x[(int64_t)b * T + i] = q;
    if (i > 0) t[(int64_t)b * T + i - 1] = q;
  }
  const int64_t fo = so / U;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < D * Tf; e += gridDim.x * blockDim.x) {
    const int d = e / Tf, j = e - d * Tf;
    const int64_t row = corpus_index(starts, offsets, n_utts, (fo + j) * U) / U;
    h[((int64_t)b * D + d) * Tf + j] = scaled_feat(feat, row * D + d, d, mean, scale, feat_f64);
  }
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_make_train_batch(const float* wave, const void* feat, const int32_t* frame_of_sample, int64_t s0,
                                 int64_t hop, int U, int64_t cap_s, int64_t cap_f, const double* mean, const double* scale,
                                 int64_t* x, int64_t* t, float* h, int B, int T, int Tf, int D, int feat_f64, int mu,
                                 void* stream) {
  WNB_REQUIRE(wave && feat && x && t && h, "make_train_batch: null pointer");
  WNB_REQUIRE(B > 0 && T > 0 && Tf > 0 && D > 0 && mu > 1 && (!mean == !scale) && s0 >= 0 && hop >= 0 && U >= 1 &&
                  cap_s > T && cap_f >= Tf,
              "make_train_batch: bad arguments");
  const int work = (T + 1 > D * Tf) ? T + 1 : D * Tf;
  dim3 grid((unsigned)((work + 255) / 256 < device_sms() ? (work + 255) / 256 : device_sms()), (unsigned)B);
  make_train_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(wave, feat, frame_of_sample, s0, hop, U, cap_s, cap_f, mean,
                                                                 scale, x, t, h, B, T, Tf, D, feat_f64, (float)(mu - 1),
                                                                 log(1.0 + (double)(mu - 1)));   // wavenet.py:27 mu = mu - 1
  WNB_CHECK_LAUNCH("make_train_batch");
  return WNB_OK;
}

WNB_API int wnb_make_train_batch_corpus(const int16_t* wave, const void* feat, const int64_t* starts, const int64_t* offsets,
                                        int n_utts, int64_t table_begin, int64_t table_end, int64_t s0, int64_t hop, int U,
                                        const double* mean, const double* scale, int64_t* x, int64_t* t, float* h, int B,
                                        int T, int Tf, int D, int feat_f64, int mu, void* stream) {
  WNB_REQUIRE(wave && feat && starts && offsets && x && t && h, "make_train_batch_corpus: null pointer");
  WNB_REQUIRE(B > 0 && T > 0 && Tf > 0 && D > 0 && mu > 1 && (!mean == !scale) && n_utts > 0 && hop >= 0 && U >= 1 &&
                  s0 >= table_begin && s0 >= 0 && table_begin <= table_end,
              "make_train_batch_corpus: bad arguments");
  const int64_t last = s0 + (int64_t)(B - 1) * hop;   // start of the last window
  WNB_REQUIRE(last + T + 1 <= table_end && (last / U + Tf - 1) * U < table_end,
              "make_train_batch_corpus: the windows reach past the end of the table");
  const int work = (T + 1 > D * Tf) ? T + 1 : D * Tf;
  dim3 grid((unsigned)((work + 255) / 256 < device_sms() ? (work + 255) / 256 : device_sms()), (unsigned)B);
  make_train_batch_corpus_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      wave, feat, starts, offsets, n_utts, s0, hop, U, mean, scale, x, t, h, B, T, Tf, D, feat_f64, (float)(mu - 1),
      log(1.0 + (double)(mu - 1)));
  WNB_CHECK_LAUNCH("make_train_batch_corpus");
  return WNB_OK;
}

}  // extern "C"
