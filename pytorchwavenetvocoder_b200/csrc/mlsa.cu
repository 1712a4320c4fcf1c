// mlsa.cu -- wnb_mlsa_filter: the reference's MLSA noise-shaping filter (bin/noise_shaping.py:46-87: pysptk
// Synthesizer(MLSADF(order, alpha), hopsize).synthesis(x, tiled coefficients)) for a BATCH of utterances on the GPU.
//
// The filter is a per-sample recursion (SPTK mlsadf: two cascaded Pade approximants of exp(), the second over a chain of
// `order` first-order all-pass sections), so one utterance is a 160 000-step dependency chain -- the parallelism is
//   * the pd (4 or 5) Pade stages of the second approximant: within one sample each stage filters the PREVIOUS sample's
//     output of the stage before it, so the stages are independent -> one lane per stage, 8 lanes per utterance;
//   * utterances: 4 per warp, one warp per block, as many blocks as the batch needs (the reference runs n_jobs CPU
//     processes over the file list, noise_shaping.py:166-187).
// Arithmetic is fp64 with the operation ORDER of the C recursion and no FMA contraction (__dmul_rn / __dadd_rn), so the
// output is bit-identical to the CPU oracle (oracle/mlsa_oracle.c, compiled -ffp-contract=off).  The all-pass chain of a
// stage keeps its state e[1..m] in shared memory; SPTK's delay-line shift d[i] = d[i-1] disappears by reading
// e_prev[i-1] where it reads the shifted d[i].  Samples move 8 at a time per utterance (one per lane, shuffled to the
// lanes as needed); int16 in / out is the wav path of the CLI (np.float64(x) in, np.int16(y) out: truncation).
// Without a state table every utterance starts from a zero filter state.  With one (wnb_mlsa_filter_state) a segment
// loads its slot's state before its first sample and stores it right after its OWN last sample: the warp runs its 4
// segments up to the longest one, so the shorter ones keep filtering zeros past their end, which the carried state must
// not see.  Chained segments therefore filter exactly what one segment holding all their samples filters.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wnb200.h"
#include "common.cuh"

namespace wnb {

__constant__ double c_pade[21] = {1.0,
                                  1.0, 0.0,
                                  1.0, 0.0, 0.0,
                                  1.0, 0.0, 0.0, 0.0,
                                  1.0, 0.4999273, 0.1067005, 0.01170221, 0.0005656279,
                                  1.0, 0.4999391, 0.1107098, 0.01369984, 0.0009564853, 0.00003041721};

// Per-segment slots of a stateful launch, passed by value: slot[u] >= 0 loads slot slot[u]; slot[u] = -1 - s starts
// slot s from a zero state.  Either way the state after the segment goes to slot s.
struct MlsaSlots {
  int slot[WNB_MLSA_MAX_STATE_SEGMENTS];
};

// State of one filter instance (wnb_mlsa_state_doubles(m, PD) doubles, include/wnb200.h): d1[1..PD], pt1[0..PD], pt20,
// pt_own of stages 1..PD, then each stage's all-pass chain e[1..m].
__host__ __device__ constexpr int mlsa_state_pt1(int pd) { return pd; }
__host__ __device__ constexpr int mlsa_state_pt20(int pd) { return 2 * pd + 1; }
__host__ __device__ constexpr int mlsa_state_own(int pd) { return 2 * pd + 2; }
__host__ __device__ constexpr int mlsa_state_chain(int pd) { return 3 * pd + 2; }

template <int PD>
__global__ void __launch_bounds__(32) mlsa_kernel(const void* __restrict__ xin, int x_i16, const long long* __restrict__ offsets,
                                                  int n_utts, const double* __restrict__ coef, int m, double a, double gain,
                                                  void* __restrict__ yout, int y_i16, double* __restrict__ states,
                                                  const __grid_constant__ MlsaSlots slots) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x, g = lane >> 3, s = lane & 7;
  const int stride = (m + 1) | 1;                 // odd number of doubles: the 16 stage lanes hit distinct banks
  double* bsh = sm;                               // b[0..m]
  double* E = sm + (m + 2) + (size_t)(g * PD + (s < PD ? s : 0)) * stride;   // this lane's all-pass chain e[1..m]
  for (int i = lane; i <= m; i += 32) bsh[i] = coef[i];
  for (int i = lane; i < 4 * PD * stride; i += 32) sm[(m + 2) + i] = 0.0;
  __syncwarp();
  const int u = blockIdx.x * 4 + g;
  const long long off = u < n_utts ? offsets[u] : 0;
  const long long len = u < n_utts ? offsets[u + 1] - off : 0;
  double* st = nullptr;     // this segment's state slot (null: zero start, nothing stored)
  bool load = false;
  if (states != nullptr && u < n_utts) {
    const int v = slots.slot[u];
    load = v >= 0;
    st = states + (size_t)(v >= 0 ? v : -1 - v) * (size_t)(mlsa_state_chain(PD) + PD * m);
  }
  long long maxlen = len;
  maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, 8));
  maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, 16));
  const double aa = __dsub_rn(1.0, __dmul_rn(a, a));
  const double* pade = &c_pade[PD * (PD + 1) / 2];
  const double b1 = bsh[1];
  // first approximant (every lane of the group carries the same copy): d1[1..PD], pt1[0..PD]
  double d1[PD + 1], pt1[PD + 1];
#pragma unroll
  for (int i = 0; i <= PD; i++) { d1[i] = 0.0; pt1[i] = 0.0; }
  double pt20 = 0.0;      // second approximant: pt[0]
  double pt_own = 0.0;    // pt[s + 1]: this stage's output for the previous sample
  if (load) {
#pragma unroll
    for (int i = 1; i <= PD; i++) d1[i] = st[i - 1];
#pragma unroll
    for (int i = 0; i <= PD; i++) pt1[i] = st[mlsa_state_pt1(PD) + i];
    pt20 = st[mlsa_state_pt20(PD)];
    if (s < PD) {
      pt_own = st[mlsa_state_own(PD) + s];
      for (int i = 1; i <= m; i++) E[i] = st[mlsa_state_chain(PD) + s * m + i - 1];   // after the zeroing's __syncwarp
    }
  }
  const int16_t* x16 = reinterpret_cast<const int16_t*>(xin);
  const double* x64 = reinterpret_cast<const double*>(xin);
  int16_t* y16 = reinterpret_cast<int16_t*>(yout);
  double* y64 = reinterpret_cast<double*>(yout);
  for (long long n0 = 0; n0 < maxlen; n0 += 8) {
    double xreg = 0.0, yreg = 0.0;
    if (n0 + s < len) xreg = x_i16 ? (double)x16[off + n0 + s] : x64[off + n0 + s];
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      double x = __dmul_rn(__shfl_sync(0xffffffffu, xreg, (g << 3) + j), gain);
      // ---- mlsadf1 ----
      double out = 0.0;
#pragma unroll
      for (int i = PD; i >= 1; i--) {
        d1[i] = __dadd_rn(__dmul_rn(aa, pt1[i - 1]), __dmul_rn(a, d1[i]));
        pt1[i] = __dmul_rn(d1[i], b1);
        const double v = __dmul_rn(pt1[i], pade[i]);
        x = (i & 1) ? __dadd_rn(x, v) : __dsub_rn(x, v);
        out = __dadd_rn(out, v);
      }
      pt1[0] = x;
      x = __dadd_rn(out, x);
      // ---- mlsadf2: stage s + 1 filters pt[s] of the previous sample through the all-pass chain (mlsafir) ----
      const double up = __shfl_up_sync(0xffffffffu, pt_own, 1, 8);
      const double in = s == 0 ? pt20 : up;
      double ys = 0.0;
      if (s < PD) {
        const double e1_old = E[1];
        const double e1 = __dadd_rn(__dmul_rn(aa, in), __dmul_rn(a, e1_old));
        E[1] = e1;
        double prev_old = e1_old, prev_new = e1;
#pragma unroll 4
        for (int i = 2; i <= m; i++) {
          const double cur_old = E[i];
          const double e = __dadd_rn(prev_old, __dmul_rn(a, __dsub_rn(cur_old, prev_new)));
          ys = __dadd_rn(ys, __dmul_rn(e, bsh[i]));
          E[i] = e;
          prev_old = cur_old;
          prev_new = e;
        }
      }
      out = 0.0;
#pragma unroll
      for (int i = PD; i >= 1; i--) {
        const double pti = __shfl_sync(0xffffffffu, ys, (g << 3) + i - 1);
        const double v = __dmul_rn(pti, pade[i]);
        x = (i & 1) ? __dadd_rn(x, v) : __dsub_rn(x, v);
        out = __dadd_rn(out, v);
      }
      pt20 = x;
      out = __dadd_rn(out, x);
      pt_own = ys;
      if (s == j) yreg = out;
      if (st != nullptr && n0 + j + 1 == len) {   // the segment's last sample: store the state it leaves
        if (s == 0) {
#pragma unroll
          for (int i = 1; i <= PD; i++) st[i - 1] = d1[i];
#pragma unroll
          for (int i = 0; i <= PD; i++) st[mlsa_state_pt1(PD) + i] = pt1[i];
          st[mlsa_state_pt20(PD)] = pt20;
        }
        if (s < PD) {
          st[mlsa_state_own(PD) + s] = pt_own;
          for (int i = 1; i <= m; i++) st[mlsa_state_chain(PD) + s * m + i - 1] = E[i];
        }
      }
    }
    if (n0 + s < len) {
      if (y_i16) y16[off + n0 + s] = (int16_t)__double2ll_rz(yreg);
      else y64[off + n0 + s] = yreg;
    }
  }
}

}  // namespace wnb

using namespace wnb;

namespace {

int mlsa_launch(const void* x, int x_is_i16, const long long* offsets, int n_utts, const double* coef, int order,
                double alpha, int pd, double gain, void* y, int y_is_i16, double* states, const MlsaSlots& slots,
                void* stream, const char* what) {
  const int stride = (order + 1) | 1;
  const size_t smem = sizeof(double) * ((size_t)(order + 2) + (size_t)4 * pd * stride);
  const unsigned grid = (unsigned)((n_utts + 3) / 4);
  cudaStream_t st = (cudaStream_t)stream;
  if (pd == 4) {
    WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(mlsa_kernel<4>), smem));
    mlsa_kernel<4><<<grid, 32, smem, st>>>(x, x_is_i16, offsets, n_utts, coef, order, alpha, gain, y, y_is_i16, states,
                                           slots);
  } else {
    WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(mlsa_kernel<5>), smem));
    mlsa_kernel<5><<<grid, 32, smem, st>>>(x, x_is_i16, offsets, n_utts, coef, order, alpha, gain, y, y_is_i16, states,
                                           slots);
  }
  WNB_CHECK_LAUNCH(what);
  return WNB_OK;
}

}  // namespace

extern "C" {

WNB_API int wnb_mlsa_filter(const void* x, int x_is_i16, const long long* offsets, int n_utts, const double* coef, int order,
                            double alpha, int pd, double gain, void* y, int y_is_i16, void* stream) {
  WNB_REQUIRE(x && offsets && coef && y, "mlsa_filter: null pointer");
  WNB_REQUIRE(n_utts > 0 && order >= 2 && order <= 255, "mlsa_filter: need n_utts > 0 and 2 <= order <= 255");
  WNB_REQUIRE(pd == 4 || pd == 5, "mlsa_filter: pd must be 4 or 5 (SPTK's Pade tables)");
  WNB_REQUIRE(alpha > -1.0 && alpha < 1.0, "mlsa_filter: |alpha| must be < 1");
  static const MlsaSlots no_slots = {};
  return mlsa_launch(x, x_is_i16, offsets, n_utts, coef, order, alpha, pd, gain, y, y_is_i16, nullptr, no_slots, stream,
                     "mlsa_filter");
}

WNB_API size_t wnb_mlsa_state_doubles(int order, int pd) {
  if (order < 2 || order > 255 || (pd != 4 && pd != 5)) return 0;
  return (size_t)mlsa_state_chain(pd) + (size_t)pd * order;
}

WNB_API int wnb_mlsa_filter_state(const void* x, int x_is_i16, const long long* offsets, int n_segs, const double* coef,
                                  int order, double alpha, int pd, double gain, void* y, int y_is_i16, double* states,
                                  int n_slots, const int32_t* slots, const int32_t* zero_start, void* stream) {
  WNB_REQUIRE(x && offsets && coef && y, "mlsa_filter_state: null pointer");
  WNB_REQUIRE(states && slots, "mlsa_filter_state: need a state table and the segments' slot indices");
  WNB_REQUIRE(n_segs > 0 && n_segs <= WNB_MLSA_MAX_STATE_SEGMENTS && order >= 2 && order <= 255,
              "mlsa_filter_state: need 0 < n_segs <= %d and 2 <= order <= 255", WNB_MLSA_MAX_STATE_SEGMENTS);
  WNB_REQUIRE(pd == 4 || pd == 5, "mlsa_filter_state: pd must be 4 or 5 (SPTK's Pade tables)");
  WNB_REQUIRE(alpha > -1.0 && alpha < 1.0, "mlsa_filter_state: |alpha| must be < 1");
  WNB_REQUIRE(n_slots > 0, "mlsa_filter_state: need n_slots > 0");
  MlsaSlots p;
  for (int u = 0; u < n_segs; u++) {
    WNB_REQUIRE(slots[u] >= 0 && slots[u] < n_slots, "mlsa_filter_state: segment %d: slot %d of %d", u, slots[u],
                n_slots);
    for (int k = 0; k < u; k++)
      WNB_REQUIRE(slots[k] != slots[u], "mlsa_filter_state: slot %d given twice", slots[u]);
    p.slot[u] = (zero_start && zero_start[u]) ? -1 - slots[u] : slots[u];
  }
  return mlsa_launch(x, x_is_i16, offsets, n_segs, coef, order, alpha, pd, gain, y, y_is_i16, states, p, stream,
                     "mlsa_filter_state");
}

}  // extern "C"
