// decode.cu -- persistent fast-generate kernel (wavenet.py:309-395 fast_generate, :397-511
// batch_fast_generate, :538-549 _generate_residual_forward).
//
// One launch generates every sample of every utterance.  A CTA owns NU utterances for their whole life:
// it steps the per-layer dilation FIFOs from the all-zero state through the padded/seed prefix
// (teacher forced, residual path only -- equivalent to the reference's warm-up convolution,
// wavenet.py:337-350) and then free-runs: front gather -> L gated blocks -> post net -> argmax /
// softmax sample, sample by sample, without ever returning to the host.
//
// Per step every matrix-vector product is a K-major GEMV: warp lanes read 512 contiguous bytes of one
// weight row (float4 per lane) and broadcast the activation from shared memory, so the weight stream
// (8.6 MB fp32 at 64/512, resident in the 50 MB L2) is perfectly coalesced; K is split over the CTA's
// warps and reduced through shared memory.  The dilation queues (786 KB fp32 per utterance at 64/512)
// live in global memory but are L2 resident; all (ks-1)*L taps of a step are prefetched at the top of
// the step because they only depend on earlier steps.  fp32 FFMA throughout: autoregressive argmax
// parity does not survive tf32/bf16 (SURVEY.md section 7).  There is no inter-CTA communication, hence
// no way to dead-lock the GPU.
#include "common.cuh"

namespace wnb {

constexpr int kDecThreads = 256;
constexpr int kMaxLayers = 64;

struct DecodeParams {
  int32_t* xs; const float* h; const float* up_w; const float* up_b;
  const float *wf, *bf, *w1d, *b1, *w2d, *b2, *wp1d, *bp1, *wp2d, *bp2;
  float* queues; const int32_t* n_samples; const float* uniforms; float* logits_out;
  int B, P, max_n, n_pad, Th, Q, A, Ap, R, S, ks, U, mode, L;
  int pos0, i0, i_last, h_last, stride_xs;   // the call's window (common.cuh DecodeWindow)
  int O1, O2, Sp, Qp;  // padded (multiple of 4) output widths of the K-major matrices
  unsigned long long seed;
  int dil[kMaxLayers];
  long long qoff[kMaxLayers];  // float offset of layer l's ring inside one utterance's queue block
  long long q_per_utt;
  int partial_pad;  // 0 .. 3 floats between qtap's end and the 16-byte aligned partial (decode_partial_offset)
};

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1, uint32_t (&out)[4]) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// partial[part][u][o] = sum_{k in part} Wt[k][o] * x[u][k]   (o in float4 columns)
template <int NU, bool RELU_X>
__device__ __forceinline__ void gemv_partial(const float* __restrict__ Wt, int ldw, int K, int O,
                                             const float* __restrict__ x, int ldx, float* __restrict__ partial,
                                             int& parts_out) {
  const int lanes = O >> 2;  // float4 columns
  const int tid = threadIdx.x;
  if (lanes <= kDecThreads) {
    const int parts = kDecThreads / lanes;
    parts_out = parts;
    const int lane = tid % lanes, part = tid / lanes;
    if (part < parts) {
      float4 acc[NU];
#pragma unroll
      for (int u = 0; u < NU; u++) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4* wp = reinterpret_cast<const float4*>(Wt) + lane;
      const int ld4 = ldw >> 2;
      int k = part;
      for (; k + 3 * parts < K; k += 4 * parts) {
        const float4 w0 = __ldg(wp + (size_t)k * ld4);
        const float4 w1 = __ldg(wp + (size_t)(k + parts) * ld4);
        const float4 w2 = __ldg(wp + (size_t)(k + 2 * parts) * ld4);
        const float4 w3 = __ldg(wp + (size_t)(k + 3 * parts) * ld4);
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float x0 = x[u * ldx + k], x1 = x[u * ldx + k + parts], x2 = x[u * ldx + k + 2 * parts],
                x3 = x[u * ldx + k + 3 * parts];
          if (RELU_X) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); x2 = fmaxf(x2, 0.f); x3 = fmaxf(x3, 0.f); }
          acc[u].x = fmaf(w0.x, x0, acc[u].x); acc[u].y = fmaf(w0.y, x0, acc[u].y);
          acc[u].z = fmaf(w0.z, x0, acc[u].z); acc[u].w = fmaf(w0.w, x0, acc[u].w);
          acc[u].x = fmaf(w1.x, x1, acc[u].x); acc[u].y = fmaf(w1.y, x1, acc[u].y);
          acc[u].z = fmaf(w1.z, x1, acc[u].z); acc[u].w = fmaf(w1.w, x1, acc[u].w);
          acc[u].x = fmaf(w2.x, x2, acc[u].x); acc[u].y = fmaf(w2.y, x2, acc[u].y);
          acc[u].z = fmaf(w2.z, x2, acc[u].z); acc[u].w = fmaf(w2.w, x2, acc[u].w);
          acc[u].x = fmaf(w3.x, x3, acc[u].x); acc[u].y = fmaf(w3.y, x3, acc[u].y);
          acc[u].z = fmaf(w3.z, x3, acc[u].z); acc[u].w = fmaf(w3.w, x3, acc[u].w);
        }
      }
      for (; k < K; k += parts) {
        const float4 w0 = __ldg(wp + (size_t)k * ld4);
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float x0 = x[u * ldx + k];
          if (RELU_X) x0 = fmaxf(x0, 0.f);
          acc[u].x = fmaf(w0.x, x0, acc[u].x); acc[u].y = fmaf(w0.y, x0, acc[u].y);
          acc[u].z = fmaf(w0.z, x0, acc[u].z); acc[u].w = fmaf(w0.w, x0, acc[u].w);
        }
      }
#pragma unroll
      for (int u = 0; u < NU; u++)
        reinterpret_cast<float4*>(partial + ((size_t)part * NU + u) * O)[lane] = acc[u];
    }
  } else {
    // very wide outputs: one part, loop over column chunks
    parts_out = 1;
    for (int lane = tid; lane < lanes; lane += kDecThreads) {
      float4 acc[NU];
#pragma unroll
      for (int u = 0; u < NU; u++) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4* wp = reinterpret_cast<const float4*>(Wt) + lane;
      const int ld4 = ldw >> 2;
      for (int k = 0; k < K; k++) {
        const float4 w0 = __ldg(wp + (size_t)k * ld4);
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float x0 = x[u * ldx + k];
          if (RELU_X) x0 = fmaxf(x0, 0.f);
          acc[u].x = fmaf(w0.x, x0, acc[u].x); acc[u].y = fmaf(w0.y, x0, acc[u].y);
          acc[u].z = fmaf(w0.z, x0, acc[u].z); acc[u].w = fmaf(w0.w, x0, acc[u].w);
        }
      }
#pragma unroll
      for (int u = 0; u < NU; u++) reinterpret_cast<float4*>(partial + (size_t)u * O)[lane] = acc[u];
    }
  }
}

__device__ __forceinline__ float reduce_parts(const float* partial, int parts, int NU, int O, int u, int o) {
  float s = 0.f;
  for (int p = 0; p < parts; p++) s += partial[((size_t)p * NU + u) * O + o];
  return s;
}

template <int NU>
__global__ void __launch_bounds__(kDecThreads) decode_kernel(const DecodeParams p) {
  extern __shared__ __align__(16) float smem[];
  const int R = p.R, S = p.S, Q = p.Q, Ap = p.Ap, ks = p.ks, L = p.L;
  const int K1 = ks * R + Ap;
  const int ntap = (ks - 1) * L;
  // shared memory carve-up (floats).  Only `partial` is accessed as float4; it starts at a multiple of 4 floats (16
  // bytes, decode_partial_offset).  The regions before it are read and written as scalars and may have any length.
  float* xcat = smem;                          // [NU][K1]
  float* cur = xcat + NU * K1;                 // [NU][R]
  float* zs = cur + NU * R;                    // [NU][R]
  float* skipacc = zs + NU * R;                // [NU][S]
  float* h1 = skipacc + NU * S;                // [NU][S]
  float* logit = h1 + NU * S;                  // [NU][Qp]
  float* hcol = logit + NU * p.Qp;             // [NU][Ap]
  float* qtap = hcol + NU * Ap;                // [NU][ntap][R]
  float* partial = qtap + (size_t)NU * ntap * R + p.partial_pad;  // [parts][NU][O]  (>= NU*max(1024, Omax))
  __shared__ int s_n[NU];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int u0 = blockIdx.x * NU;
  const int stride_xs = p.stride_xs;

  if (tid < NU) s_n[tid] = (u0 + tid < p.B) ? p.i0 + p.n_samples[u0 + tid] : 0;   // absolute end
  __syncthreads();
  int nmax = 0;
#pragma unroll
  for (int u = 0; u < NU; u++) nmax = max(nmax, s_n[u]);
  if (nmax <= p.i0) return;
  const int last_pos = p.P - 1 + nmax - 1;

  for (int pos = p.pos0; pos <= last_pos; pos++) {
    const bool want = pos >= p.P - 1;  // free-running: need logits
    // ---- stage 0: front gather, aux column, queue-tap prefetch ----
    for (int e = tid; e < NU * R; e += kDecThreads) {
      const int u = e / R, r = e - u * R;
      const int ug = min(u0 + u, p.B - 1);
      float v = __ldg(p.bf + r);
      for (int k = 0; k < ks; k++) {
        const int pp = pos - (ks - 1 - k);
        if (pp >= 0) {
          int q = p.xs[(size_t)ug * stride_xs + pp] % Q;
          if (q < 0) q += Q;
          v += __ldg(p.wf + ((size_t)k * Q + q) * R + r);
        }
      }
      cur[e] = v;
    }
    for (int e = tid; e < NU * Ap; e += kDecThreads) {
      const int u = e / Ap, a = e - u * Ap;
      const int ug = min(u0 + u, p.B - 1);
      float v = 0.f;
      if (a < p.A) {
        const int j = max(pos - p.n_pad, 0);
        if (p.U > 0) {
          const int tf = min(j / p.U, p.h_last), jj = j % p.U;
          v = fmaf(__ldg(p.h + ((size_t)ug * p.A + a) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
        } else {
          v = __ldg(p.h + ((size_t)ug * p.A + a) * p.Th + min(j, p.h_last));
        }
      }
      hcol[e] = v;
    }
    for (int e = tid; e < NU * ntap * R; e += kDecThreads) {
      const int r = e % R;
      const int tp = (e / R) % ntap;
      const int u = e / (R * ntap);
      const int ug = min(u0 + u, p.B - 1);
      const int l = tp / (ks - 1), j = tp - l * (ks - 1);  // tap j (0 = oldest)
      const int d = p.dil[l];
      const int s = (ks - 1 - j) * d;
      float v = 0.f;
      if (pos - s >= 0) {
        const int qlen = (ks - 1) * d;
        const float* q = p.queues + (size_t)ug * p.q_per_utt + p.qoff[l];
        v = __ldcg(q + (size_t)((pos - s) % qlen) * R + r);
      }
      qtap[e] = v;
    }
    __syncthreads();

    for (int l = 0; l < L; l++) {
      // ---- build xcat = [taps | cur | aux] and push cur into the ring ----
      const int d = p.dil[l];
      for (int e = tid; e < NU * K1; e += kDecThreads) {
        const int u = e / K1, k = e - u * K1;
        float v;
        if (k < (ks - 1) * R) {
          const int j = k / R, r = k - j * R;
          v = qtap[((size_t)u * ntap + l * (ks - 1) + j) * R + r];
        } else if (k < ks * R) {
          v = cur[u * R + (k - (ks - 1) * R)];
        } else {
          v = hcol[u * Ap + (k - ks * R)];
        }
        xcat[e] = v;
      }
      if (ks > 1) {
        const int qlen = (ks - 1) * d;
        for (int e = tid; e < NU * R; e += kDecThreads) {
          const int u = e / R, r = e - u * R;
          if (u0 + u < p.B) {
            float* q = p.queues + (size_t)(u0 + u) * p.q_per_utt + p.qoff[l];
            __stcg(q + (size_t)(pos % qlen) * R + r, cur[e]);
          }
        }
      }
      __syncthreads();
      int parts;
      gemv_partial<NU, false>(p.w1d + (size_t)l * K1 * p.O1, p.O1, K1, p.O1, xcat, K1, partial, parts);
      __syncthreads();
      for (int e = tid; e < NU * R; e += kDecThreads) {
        const int u = e / R, c = e - u * R;
        const float a = reduce_parts(partial, parts, NU, p.O1, u, c) + __ldg(p.b1 + (size_t)l * 2 * R + c);
        const float g = reduce_parts(partial, parts, NU, p.O1, u, R + c) + __ldg(p.b1 + (size_t)l * 2 * R + R + c);
        zs[e] = sigmoidf_(a) * tanhf(g);
      }
      __syncthreads();
      const int O2 = want ? p.O2 : ((R + 3) & ~3);
      gemv_partial<NU, false>(p.w2d + (size_t)l * R * p.O2, p.O2, R, O2, zs, R, partial, parts);
      __syncthreads();
      const int nout = want ? (R + S) : R;
      for (int e = tid; e < NU * nout; e += kDecThreads) {
        const int u = e / nout, o = e - u * nout;
        const float v = reduce_parts(partial, parts, NU, O2, u, o) + __ldg(p.b2 + (size_t)l * (R + S) + o);
        if (o < R) {
          cur[u * R + o] += v;
        } else {
          float* dst = skipacc + u * S + (o - R);
          *dst = (l == 0) ? v : (*dst + v);  // python `0 + s0 + s1 ...`, wavenet.py:374
        }
      }
      __syncthreads();
    }

    if (want) {
      int parts;
      gemv_partial<NU, true>(p.wp1d, p.Sp, S, p.Sp, skipacc, S, partial, parts);
      __syncthreads();
      for (int e = tid; e < NU * S; e += kDecThreads) {
        const int u = e / S, o = e - u * S;
        h1[e] = fmaxf(reduce_parts(partial, parts, NU, p.Sp, u, o) + __ldg(p.bp1 + o), 0.f);
      }
      __syncthreads();
      gemv_partial<NU, false>(p.wp2d, p.Qp, S, p.Qp, h1, S, partial, parts);
      __syncthreads();
      const int i = pos - (p.P - 1);  // index of the sample being generated
      for (int e = tid; e < NU * Q; e += kDecThreads) {
        const int u = e / Q, o = e - u * Q;
        const float v = reduce_parts(partial, parts, NU, p.Qp, u, o) + __ldg(p.bp2 + o);
        logit[u * p.Qp + o] = v;
        if (p.logits_out && u0 + u < p.B && i < s_n[u])
          p.logits_out[((size_t)(u0 + u) * p.max_n + i) * Q + o] = v;
      }
      __syncthreads();
      // ---- pick: warp u handles utterance u ----
      if (warp < NU) {
        const int u = warp;
        const float* lg = logit + u * p.Qp;
        const int chunk = (Q + 31) / 32;
        const int q0 = lane * chunk, q1 = min(q0 + chunk, Q);
        float best = -INFINITY;
        int bi = 0x7fffffff;
        for (int q = q0; q < q1; q++)
          if (lg[q] > best) { best = lg[q]; bi = q; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        int pick = bi;  // first maximum (torch CPU argmax semantics)
        if (p.mode == WNB_MODE_SAMPLING) {
          // inverse-CDF draw from softmax(logits)  (wavenet.py:377-379 uses torch Categorical)
          float uni;
          if (p.uniforms) {
            uni = p.uniforms[(size_t)min(u0 + u, p.B - 1) * p.max_n + min(i, p.i_last)];
          } else {
            uint32_t r[4];
            philox4x32_10((uint32_t)i, (uint32_t)(u0 + u), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), r);
            uni = (float)(r[0] >> 8) * (1.0f / 16777216.0f);
          }
          float lsum = 0.f;
          int lnz = -1;
          for (int q = q0; q < q1; q++) {
            const float e = expf(lg[q] - best);
            lsum += e;
            if (e > 0.f) lnz = q;
          }
          float incl = lsum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          pick = sample_pick(incl, lsum, lnz, uni, lane, [&](float start, float target) {   // (common.cuh)
            float c = start;
            for (int q = q0; q < q1; q++) {
              const float e = expf(lg[q] - best);
              c += e;
              if (c > target && e > 0.f) return q;
            }
            return -1;
          });
        }
        if (lane == 0 && u0 + u < p.B && i < s_n[u]) p.xs[(size_t)(u0 + u) * stride_xs + pos + 1] = pick;
      }
      __syncthreads();
    }
  }
}

// decode_kernel's shared-memory carve-up, in floats: the scalar regions xcat .. qtap, then `partial`.
// gemv_partial stores float4 at partial + (part * NU + u) * O with O a multiple of 4, so partial must start at a
// multiple of 4 floats (16 bytes) from the 16-byte aligned base.  R and S need not be multiples of 4 on this kernel,
// so the scalar regions can end at 2 or 3 mod 4 floats (Q 256, Ap 32, R 6, S 8, ks 2, L 3 gives 378 at NU 1).
// partial's offset is rounded up to 4 floats and the kernel skips the difference (DecodeParams::partial_pad); the
// launcher sizes shared memory from the same offset.
static size_t decode_scalar_floats(int NU, int R, int S, int Qp, int Ap, int ks, int L) {
  const size_t K1 = (size_t)ks * R + Ap;
  return (size_t)NU * (K1 + 2 * (size_t)R + 2 * (size_t)S + Qp + Ap + (size_t)(ks - 1) * L * R);
}
static size_t decode_partial_offset(int NU, int R, int S, int Qp, int Ap, int ks, int L) {
  return (decode_scalar_floats(NU, R, S, Qp, Ap, ks, L) + 3) & ~(size_t)3;
}

static size_t decode_smem_floats(int NU, int R, int S, int Qp, int Ap, int ks, int L, int O1, int O2, int Sp) {
  size_t omax = (size_t)O1;
  if ((size_t)O2 > omax) omax = O2;
  if ((size_t)Sp > omax) omax = Sp;
  if ((size_t)Qp > omax) omax = Qp;
  if (omax < 1024) omax = 1024;
  return decode_partial_offset(NU, R, S, Qp, Ap, ks, L) + (size_t)NU * omax;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API size_t wnb_decode_workspace(int B, int R, int ks, const int32_t* host_dilations, int L) {
  size_t per = 0;
  for (int l = 0; l < L; l++) per += (size_t)(ks - 1) * host_dilations[l] * R;
  return per * sizeof(float) * (size_t)B;
}

WNB_API int wnb_decode_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                          const float* bf, const float* w1d, const float* b1, const float* w2d, const float* b2,
                          const float* wp1d, const float* bp1, const float* wp2d, const float* bp2,
                          const int32_t* host_dilations, int L, void* queues, const int32_t* n_samples,
                          const float* uniforms, float* logits_out, int B, int P, int max_n, int n_pad, int Th, int Q,
                          int A, int Ap, int R, int S, int ks, int U, int mode, uint64_t seed, int pos0, int xs_base,
                          int h_frame0, void* stream) {
  WNB_REQUIRE(B > 0 && P >= 1 && max_n >= 1 && Th >= 1 && Q > 0 && A > 0 && Ap >= A && R > 0 && S > 0 && ks >= 1 &&
                  U >= 0 && L >= 1, "decode: bad shape");
  WNB_REQUIRE(L <= kMaxLayers, "decode: more than %d layers", kMaxLayers);
  WNB_REQUIRE(xs && h && wf && bf && w1d && b1 && w2d && b2 && wp1d && bp1 && wp2d && bp2 && n_samples &&
                  (queues || ks == 1), "decode: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode: U>0 needs upsampling weight and bias");
  WNB_REQUIRE(mode == WNB_MODE_ARGMAX || mode == WNB_MODE_SAMPLING, "decode: mode should be sampling or argmax");
  WNB_REQUIRE(Ap % 4 == 0, "decode: Ap must be a multiple of 4");
  DecodeParams p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf; p.w1d = w1d; p.b1 = b1; p.w2d = w2d;
  p.b2 = b2; p.wp1d = wp1d; p.bp1 = bp1; p.wp2d = wp2d; p.bp2 = bp2; p.queues = (float*)queues;
  p.n_samples = n_samples; p.uniforms = uniforms; p.logits_out = logits_out;
  p.B = B; p.P = P; p.max_n = max_n; p.n_pad = n_pad; p.Th = Th; p.Q = Q; p.A = A; p.Ap = Ap; p.R = R; p.S = S;
  p.ks = ks; p.U = U; p.mode = mode; p.L = L; p.seed = seed;
  DecodeWindow win;
  if (!decode_window("decode", P, n_pad, U, ks, max_n, Th, pos0, xs_base, h_frame0, &win)) return WNB_ERR_INVALID;
  p.pos0 = win.pos0; p.i0 = win.i0; p.i_last = win.i_last; p.h_last = win.h_last; p.stride_xs = win.stride_xs;
  p.xs = shift_ptr(xs, -(long long)xs_base); p.h = shift_ptr(h, -(long long)h_frame0);
  p.uniforms = shift_ptr(uniforms, -(long long)win.i0); p.logits_out = shift_ptr(logits_out, -(long long)win.i0 * Q);
  p.O1 = (2 * R + 3) & ~3; p.O2 = (R + S + 3) & ~3; p.Sp = (S + 3) & ~3; p.Qp = (Q + 3) & ~3;
  long long off = 0;
  for (int l = 0; l < L; l++) {
    p.dil[l] = host_dilations[l];
    p.qoff[l] = off;
    off += (long long)(ks - 1) * host_dilations[l] * R;
  }
  p.q_per_utt = off;

  // utterances per CTA: share the weight stream between utterances once there are more utterances than
  // SMs; stay at 1 while B <= the SM count so that every utterance gets its own SM's L2 port.
  int NU = 1;
  if (B > device_sms() * 2) NU = 4; else if (B > device_sms()) NU = 2;
  size_t smem = 0;
  for (;;) {
    smem = decode_smem_floats(NU, R, S, p.Qp, Ap, ks, L, p.O1, p.O2, p.Sp) * sizeof(float);
    if (smem <= 220 * 1024 || NU == 1) break;
    NU >>= 1;
  }
  WNB_REQUIRE(smem <= 227 * 1024, "decode: configuration needs %zu bytes of shared memory per CTA", smem);
  p.partial_pad =
      (int)(decode_partial_offset(NU, R, S, p.Qp, Ap, ks, L) - decode_scalar_floats(NU, R, S, p.Qp, Ap, ks, L));
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = cdiv(B, NU);
#define WNB_LAUNCH_DECODE(N)                                                                                  \
  do {                                                                                                        \
    WNB_CUDA(cudaFuncSetAttribute(decode_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    decode_kernel<N><<<grid, kDecThreads, smem, st>>>(p);                                                     \
  } while (0)
  if (NU == 4) WNB_LAUNCH_DECODE(4);
  else if (NU == 2) WNB_LAUNCH_DECODE(2);
  else WNB_LAUNCH_DECODE(1);
#undef WNB_LAUNCH_DECODE
  WNB_CHECK_LAUNCH("decode");
  return WNB_OK;
}

}  // extern "C"
