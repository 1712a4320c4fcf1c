// melspc_stream.cu -- wnb_melspc_stream: the log mel-spectrogram of signals that arrive in chunks, bit-identical to
// wnb_melspc_lowcut + wnb_melspc over each whole signal (DESIGN.md §6 row f7).
//
// A call advances up to WNB_MELSPC_MAX_STREAM_SEGMENTS keyed signals by one chunk each and writes every frame no later
// sample can change.  Which frames those are, and which filtered samples pending frames still read (the carry), is host
// arithmetic (utils/melspc.py melspc_frames_ready / melspc_carry_start): the kernels only follow the segment table.
//
// Slot state (wnb_melspc_stream_state_doubles): the last n_taps - 1 input samples (the FIR history; zeros for a new
// key), then the carry: filtered samples [cs, n) of a signal that has had n samples, cs = melspc_carry_start(n), at most
// fftl - 1 of them.
//
// Two launches, and the carry hazard.  A call reads each slot's old carry and history and stores new ones; a block of
// the same launch must never read a slot another block has overwritten.  So the first launch (stream_prep_kernel) only
// reads slots: per segment it writes a scratch region [old carry | filtered chunk | new history].  The second
// (stream_frames_kernel) only reads scratch: one block per frame, plus one block per segment that copies the new carry
// and history from scratch into the slot.  No block reads a slot after the first launch, so the stores cannot race.
//
// The FIR is lowcut_fma over [history | chunk] and each frame is melspc_frame over the scratch region, the device
// functions the whole-file kernels run (melspc_frame.cuh), so every value is computed by the same instructions in the
// same order.  No atomics: two runs are bit-identical.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wnb200.h"
#include "common.cuh"
#include "melspc_frame.cuh"

namespace wnb {

constexpr int MSS_TILE = 1024;     // prep outputs per block
constexpr int MSS_THREADS = 256;
constexpr int MSS_FRAME_THREADS_MAX = 256;

enum { SEG_SLOT = WNB_MELSPC_SEG_SLOT, SEG_FLAGS = WNB_MELSPC_SEG_FLAGS, SEG_X_OFF = WNB_MELSPC_SEG_X_OFF,
       SEG_X_LEN = WNB_MELSPC_SEG_X_LEN, SEG_N0 = WNB_MELSPC_SEG_N_BEFORE, SEG_CS0 = WNB_MELSPC_SEG_CARRY0,
       SEG_SCRATCH = WNB_MELSPC_SEG_SCRATCH, SEG_R0 = WNB_MELSPC_SEG_R0, SEG_R1 = WNB_MELSPC_SEG_R1,
       SEG_ROW = WNB_MELSPC_SEG_OUT_ROW, SEG_CS1 = WNB_MELSPC_SEG_CARRY1, SEG_F = WNB_MELSPC_SEG_FIELDS };

__device__ __forceinline__ bool seg_has_work(const long long* d) {
  return d[SEG_R1] > d[SEG_R0] || (d[SEG_FLAGS] & WNB_MELSPC_SEG_STORE);
}

// Block (x, u): outputs [x MSS_TILE, (x + 1) MSS_TILE) of segment u's filtered chunk, the same slice of its old carry,
// and (x = 0) its new history.
__global__ void __launch_bounds__(MSS_THREADS) stream_prep_kernel(const void* __restrict__ xin, int x_i16,
                                                                  const long long* __restrict__ segs,
                                                                  const double* __restrict__ taps, int n_taps,
                                                                  const double* __restrict__ states, long long sd,
                                                                  double* __restrict__ scratch) {
  extern __shared__ double sm[];
  const long long* d = segs + (size_t)blockIdx.y * SEG_F;
  if (!seg_has_work(d)) return;
  const int H = n_taps > 0 ? n_taps - 1 : 0;
  const bool fresh = d[SEG_FLAGS] & WNB_MELSPC_SEG_NEW;
  const long long m = d[SEG_X_LEN], c = d[SEG_N0] - d[SEG_CS0];
  const double* hist = states + (size_t)d[SEG_SLOT] * sd;
  const double* carry = hist + H;
  double* out = scratch + d[SEG_SCRATCH];
  const int16_t* x16 = reinterpret_cast<const int16_t*>(xin) + d[SEG_X_OFF];
  const double* x64 = reinterpret_cast<const double*>(xin) + d[SEG_X_OFF];
  const long long tile0 = (long long)blockIdx.x * MSS_TILE;
  for (long long i = tile0 + threadIdx.x; i < c && i < tile0 + MSS_TILE; i += MSS_THREADS) out[i] = carry[i];
  // [history | chunk] at chunk index q (q < 0: history, zeros for a new key, like x[< 0] = 0 of the whole signal)
  auto raw = [&](long long q) -> double {
    if (q >= 0) return x_i16 ? (double)x16[q] : x64[q];
    return fresh ? 0.0 : hist[H + q];
  };
  if (blockIdx.x == 0 && (d[SEG_FLAGS] & WNB_MELSPC_SEG_STORE))
    for (int j = threadIdx.x; j < H; j += MSS_THREADS) out[c + m + j] = raw(m - H + j);
  if (tile0 >= m) return;
  if (n_taps == 0) {
    for (long long i = tile0 + threadIdx.x; i < m && i < tile0 + MSS_TILE; i += MSS_THREADS) out[c + i] = raw(i);
    return;
  }
  double* b = sm;                         // taps[0 .. n_taps)
  double* xs = sm + n_taps;               // [history | chunk] at tile0 - H + i, i < MSS_TILE + H
  for (int i = threadIdx.x; i < n_taps; i += MSS_THREADS) b[i] = taps[i];
  for (int i = threadIdx.x; i < MSS_TILE + H; i += MSS_THREADS) {
    const long long q = tile0 - H + i;
    xs[i] = q < m ? raw(q) : 0.0;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < MSS_TILE; r += MSS_THREADS) {
    if (tile0 + r >= m) break;
    out[c + tile0 + r] = lowcut_fma(b, n_taps, xs + r + H);
  }
}

// Blocks f < n_frames: frame f of the call (segment u: the last with segs[u][ROW] <= f).  Blocks n_frames + u: store
// segment u's new carry and history.
__global__ void __launch_bounds__(MSS_FRAME_THREADS_MAX) stream_frames_kernel(
    const long long* __restrict__ segs, int n_segs, long long n_frames, int fftl, int log2n, int hop,
    const double* __restrict__ window, const double* __restrict__ twiddles, const float* __restrict__ mel_basis,
    const int32_t* __restrict__ mel_lo, const int32_t* __restrict__ mel_hi, int n_mels, int n_taps,
    double* __restrict__ states, long long sd, const double* __restrict__ scratch, float* __restrict__ out,
    const double* __restrict__ mean, const double* __restrict__ scale, int scaler_mode, float* __restrict__ aux) {
  extern __shared__ double sm[];
  const long long f = blockIdx.x;
  if (f >= n_frames) {
    const long long* d = segs + (size_t)(f - n_frames) * SEG_F;
    if (!(d[SEG_FLAGS] & WNB_MELSPC_SEG_STORE)) return;
    const int H = n_taps > 0 ? n_taps - 1 : 0;
    const long long m = d[SEG_X_LEN], c = d[SEG_N0] - d[SEG_CS0];
    const long long keep0 = d[SEG_CS1] - d[SEG_CS0], keep = d[SEG_N0] + m - d[SEG_CS1];
    const double* src = scratch + d[SEG_SCRATCH];
    double* st = states + (size_t)d[SEG_SLOT] * sd;
    for (int j = threadIdx.x; j < H; j += blockDim.x) st[j] = src[c + m + j];
    for (long long i = threadIdx.x; i < keep; i += blockDim.x) st[H + i] = src[keep0 + i];
    return;
  }
  int lo = 0, hi = n_segs;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (segs[(size_t)mid * SEG_F + SEG_ROW] <= f) lo = mid; else hi = mid;
  }
  const long long* d = segs + (size_t)lo * SEG_F;
  const long long row0 = d[SEG_ROW], nf = d[SEG_R1] - d[SEG_R0];
  const long long t = d[SEG_R0] + (f - row0);
  const long long n_cur = d[SEG_N0] + d[SEG_X_LEN], base = d[SEG_CS0];
  const long long start = t * hop - (fftl >> 1);
  const double* src = scratch + d[SEG_SCRATCH];
  float* a = aux ? aux + (size_t)row0 * n_mels + (f - row0) : nullptr;   // (n_mels, nf) block of the segment
  double* re = sm;
  double* im = sm + fftl;
  double* re2 = sm + 2 * fftl;
  double* im2 = sm + 3 * fftl;
  melspc_frame(
      [&](int n) { return src[reflect_index(start + n, n_cur) - base]; },
      [&](int m, float v) {
        out[(size_t)f * n_mels + m] = v;
        if (a == nullptr) return;
        float s;
        if (scaler_mode == 0) {   // float64 subtract, round, float64 divide, round
          const float dv = __double2float_rn(__dsub_rn((double)v, mean[m]));
          s = __double2float_rn(__ddiv_rn((double)dv, scale[m]));
        } else {                  // float32 subtract and divide with float32 mean and scale
          s = __fdiv_rn(__fsub_rn(v, __double2float_rn(mean[m])), __double2float_rn(scale[m]));
        }
        a[(size_t)m * nf] = s;
      },
      re, im, re2, im2, fftl, (fftl >> 1) + 1, log2n, window, twiddles, mel_basis, mel_lo, mel_hi, n_mels);
}

static int fftl_log2(int fftl) {
  int log2n = 0;
  while ((1 << log2n) < fftl && log2n < 30) log2n++;
  if (fftl < WNB_MELSPC_MIN_FFTL || fftl > WNB_MELSPC_MAX_FFTL || (1 << log2n) != fftl) return -1;
  return log2n;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API size_t wnb_melspc_stream_state_doubles(int fftl, int n_taps) {
  if (fftl_log2(fftl) < 0 || n_taps < 0 || n_taps > WNB_MELSPC_MAX_TAPS) return 0;
  return (size_t)(n_taps > 0 ? n_taps - 1 : 0) + (size_t)fftl - 1;
}

WNB_API int wnb_melspc_stream(const void* x, int x_is_i16, int n_segs, const long long* segs, const long long* segs_dev,
                              long long n_frames, int fftl, int hop, const double* taps, int n_taps,
                              const double* window, const double* twiddles, const float* mel_basis,
                              const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, double* states, int n_slots,
                              double* scratch, long long scratch_doubles, float* out, const double* mean,
                              const double* scale, int scaler_mode, float* aux, void* stream) {
  WNB_REQUIRE(segs && segs_dev && states, "melspc_stream: null pointer (segment tables or state table)");
  WNB_REQUIRE(n_segs > 0 && n_segs <= WNB_MELSPC_MAX_STREAM_SEGMENTS, "melspc_stream: need 0 < n_segs <= %d, got %d",
              WNB_MELSPC_MAX_STREAM_SEGMENTS, n_segs);
  WNB_REQUIRE(hop > 0 && n_mels > 0 && n_slots > 0,
              "melspc_stream: need hop > 0, n_mels > 0 and n_slots > 0 (hop %d, n_mels %d, n_slots %d)", hop, n_mels,
              n_slots);
  WNB_REQUIRE(n_taps >= 0 && n_taps <= WNB_MELSPC_MAX_TAPS && (n_taps == 0 || taps),
              "melspc_stream: need 0 <= n_taps <= %d and taps when n_taps > 0, got %d", WNB_MELSPC_MAX_TAPS, n_taps);
  WNB_REQUIRE(scaler_mode == 0 || scaler_mode == 2, "melspc_stream: scaler_mode must be 0 or 2, got %d", scaler_mode);
  WNB_REQUIRE(!aux || (mean && scale), "melspc_stream: scaled output needs mean and scale");
  const int log2n = fftl_log2(fftl);
  if (log2n < 0) {
    set_error("melspc_stream: fftl %d is not supported (powers of two from %d to %d)", fftl, WNB_MELSPC_MIN_FFTL,
              WNB_MELSPC_MAX_FFTL);
    return WNB_ERR_UNSUPPORTED;
  }
  const long long H = n_taps > 0 ? n_taps - 1 : 0;
  long long rows = 0, max_tiles = 0, samples = 0;
  bool work = false;
  for (int u = 0; u < n_segs; u++) {
    const long long* d = segs + (size_t)u * SEG_F;
    const long long slot = d[SEG_SLOT], flags = d[SEG_FLAGS], m = d[SEG_X_LEN], n0 = d[SEG_N0], cs0 = d[SEG_CS0];
    const long long r0 = d[SEG_R0], r1 = d[SEG_R1], cs1 = d[SEG_CS1];
    WNB_REQUIRE(slot >= 0 && slot < n_slots, "melspc_stream: segment %d: slot %lld of %d", u, slot, n_slots);
    for (int k = 0; k < u; k++)
      WNB_REQUIRE(segs[(size_t)k * SEG_F + SEG_SLOT] != slot, "melspc_stream: slot %lld given twice", slot);
    WNB_REQUIRE(flags >= 0 && flags <= (WNB_MELSPC_SEG_NEW | WNB_MELSPC_SEG_STORE),
                "melspc_stream: segment %d: bad flags %lld", u, flags);
    WNB_REQUIRE(m >= 0 && d[SEG_X_OFF] >= 0 && n0 >= 0 && cs0 >= 0 && cs0 <= n0 && n0 - cs0 <= fftl - 1 &&
                    ((flags & WNB_MELSPC_SEG_NEW) != 0) == (n0 == 0),
                "melspc_stream: segment %d: bad counts (chunk %lld, before %lld, carry from %lld)", u, m, n0, cs0);
    WNB_REQUIRE(r0 >= 0 && r1 >= r0 && (r1 == r0 || n0 + m >= 1) && r1 <= 1 + (n0 + m) / hop && d[SEG_ROW] == rows,
                "melspc_stream: segment %d: bad frame range [%lld, %lld) at row %lld", u, r0, r1, d[SEG_ROW]);
    const bool store = flags & WNB_MELSPC_SEG_STORE;
    WNB_REQUIRE(!store || (cs1 >= cs0 && cs1 <= n0 + m && n0 + m - cs1 <= fftl - 1),
                "melspc_stream: segment %d: bad new carry start %lld", u, cs1);
    const bool seg_work = r1 > r0 || store;
    if (seg_work) {
      const long long need = (n0 - cs0) + m + (store ? H : 0);
      WNB_REQUIRE(scratch && d[SEG_SCRATCH] >= 0 && d[SEG_SCRATCH] + need <= scratch_doubles,
                  "melspc_stream: segment %d: scratch [%lld, +%lld) outside %lld doubles", u, d[SEG_SCRATCH], need,
                  scratch_doubles);
      const long long span = (n0 - cs0) > m ? (n0 - cs0) : m;
      const long long tiles = (span + MSS_TILE - 1) / MSS_TILE;
      max_tiles = tiles > max_tiles ? tiles : max_tiles;
      samples += m;
      work = true;
    }
    rows += r1 - r0;
  }
  WNB_REQUIRE(rows == n_frames, "melspc_stream: n_frames %lld, the segments hold %lld", n_frames, rows);
  WNB_REQUIRE(samples == 0 || x, "melspc_stream: null pointer (samples)");
  WNB_REQUIRE(n_frames == 0 || (window && twiddles && mel_basis && mel_lo && mel_hi && out),
              "melspc_stream: null pointer (tables or output)");
  if (!work) return WNB_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  const long long sd = (long long)wnb_melspc_stream_state_doubles(fftl, n_taps);
  const size_t smem1 = sizeof(double) * ((size_t)n_taps + MSS_TILE + H);
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(stream_prep_kernel), smem1));
  const dim3 grid1((unsigned)(max_tiles > 0 ? max_tiles : 1), (unsigned)n_segs);
  stream_prep_kernel<<<grid1, MSS_THREADS, smem1, st>>>(x, x_is_i16, segs_dev, taps, n_taps, states, sd, scratch);
  WNB_CHECK_LAUNCH("melspc_stream (prep)");
  const size_t smem2 = sizeof(double) * 4 * (size_t)fftl;
  const int threads = fftl / 2 < MSS_FRAME_THREADS_MAX ? fftl / 2 : MSS_FRAME_THREADS_MAX;
  WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(stream_frames_kernel), smem2));
  stream_frames_kernel<<<(unsigned)(n_frames + n_segs), threads, smem2, st>>>(
      segs_dev, n_segs, n_frames, fftl, log2n, hop, window, twiddles, mel_basis, mel_lo, mel_hi, n_mels, n_taps, states,
      sd, scratch, out, mean, scale, scaler_mode, aux);
  WNB_CHECK_LAUNCH("melspc_stream (frames)");
  return WNB_OK;
}

}  // extern "C"
