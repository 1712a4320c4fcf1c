// decode_stream_prefill.cu -- the teacher-forced warm-up of decode_stream_kernel (padded positions 0 .. P - 2), computed
// in parallel over time and bit-identical to the sequential warm-up.
//
// As in decode_prefill.cu: every x_l(t) with t < P - 1 depends only on the seed prefix, the aux features and the weights,
// and what the free-running steps need from the warm-up is the dilation queues, layer l's ring holding x_l(t) for
// t in [P - 1 - (ks - 1) d_l, P - 2].  A front kernel computes x_0, then one launch per layer l < L - 1 computes x_{l+1}
// on layer l+1's pruned window (wnb_decode_prefill_windows(dil, L, ks)), so the work does not grow with the prompt.  Queue
// slots are written for t >= max(0, P - 1 - (ks - 1) d_l) only: the slots the sequential warm-up leaves untouched stay
// untouched.  Batches larger than kRows run in groups of kRows, so the scratch (wnb_decode_prefill_workspace) is bounded.
//
// The gate and residual matrices are read from the streaming decoder's own packed buffer (_decode_stream_pack: per layer
// W1d [K1][O1] and W2res [R][Or], K-major), so row k means what it means to the decoder.
//
// Bit identity.  decode_stream_kernel's per-element arithmetic does not depend on NU; this file restates it:
//   * front: v = bf[r], then v += wf[k][q] for k = 0 .. ks - 1 (pp < 0 skipped), q = xs % Q with the negative fix-up;
//   * aux column, j = max(pos - n_pad, 0): U > 0: fmaf(h[min(j / U, h_last)], up_w[j % U], up_b); U = 0:
//     h[min(j, h_last)]; zero for a >= A;
//   * taps are zero before position 0; the K1 input is [taps j = 0 .. ks - 2 (oldest first) | x(t) | aux];
//   * every pre-activation follows consume_segment over a K x O matrix: parts = parts_for(O), chunks of
//     rows_per_chunk(O, parts) rows; in each chunk part p puts rows p, p + 2 parts, ... into acc0 and p + parts,
//     p + 3 parts, ... into acc1 (fmaf; a lone tail row lands in acc0, which the rule "row = p mod 2 parts" covers), the
//     accumulators running on across chunks; part = acc0 + acc1; then s = 0.f, s += part_p in p order (reduce_parts_s),
//     then + bias as a separate add.  Within a part the two chains are independent, so here each chain runs whole, one
//     after the other;
//   * gate: z = sigmoidf_(a) * tanhf(g) (common.cuh, same build flags); residual: x_{l+1} = x_l + (sum + b2).
#include "common.cuh"

namespace wnb {
namespace dsp {

constexpr int kChunkBytes = 32 * 1024;   // decode_stream.cu's ring chunk
constexpr int kConsThreads = 256;        // decode_stream.cu's consumer threads
constexpr int kMaxL = 64;
constexpr int kRows = 64;                // utterances per group (scratch bound)
constexpr int kThreads = 256;
constexpr int kTP = 16;                  // positions per CTA
constexpr int kKB = 32;                  // matrix rows per shared-memory stage
constexpr int kCB = 128;                 // output columns per pass (gate: 128 sigmoid + 128 tanh columns)

struct Params {
  const int32_t* xs; const float *h, *up_w, *up_b, *wf, *bf, *stream, *b1, *b2;
  float* queues;
  int B, P, n_pad, Th, Q, A, R, S, ks, U, L;
  int O1, Or, K1;
  long long layer_stride, off_w2res;
  int base, nw;              // scratch x_l: [B][R][nw], column c = position base + c
  long long q_per_utt;
  int dil[kMaxL];
  long long qoff[kMaxL];
  int lo[kMaxL];             // first position of layer l's input window: max(0, P - 1 - S_l)
};

// decode_stream.cu's consume_segment split (same integer rule)
__host__ __device__ inline int parts_for(int O) {
  const int lanes = O >> 2;
  return lanes >= kConsThreads ? 1 : kConsThreads / lanes;
}
__host__ __device__ inline int rows_per_chunk(int O, int parts) {
  int r = kChunkBytes / (O * 4);
  if (r > parts) r = (r / parts) * parts;
  return r < 1 ? 1 : r;
}

// One accumulation chain of consume_segment: the rows k = k0 + off + 2 parts i (k0 a chunk start, k - k0 < chunk rows),
// ascending, off = p + c parts for part p and accumulator c.  The partial last chunk holds a prefix of the full pattern.
struct Chain {
  int off, per, rpc, step, n;
  __device__ __forceinline__ Chain(int K, int rpc_, int parts, int off_) : off(off_), rpc(rpc_), step(2 * parts) {
    per = off < rpc ? (rpc - off + step - 1) / step : 0;
    const int rem = K % rpc;
    n = (K / rpc) * per + (off < rem ? (rem - off + step - 1) / step : 0);
  }
  __device__ __forceinline__ int row(int m) const { return (m / per) * rpc + off + (m % per) * step; }
};

// x_0(t) = the decoder's front expression, for t in [lo[0], P - 2]
__global__ void stream_prefill_front_kernel(const Params p, float* x0) {
  const int n = p.P - 1 - p.lo[0], R = p.R, Q = p.Q, ks = p.ks;
  const long long total = (long long)p.B * R * n;
  const int qlen = (ks - 1) * p.dil[0];
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % n);
    const long long br = e / n;
    const int r = (int)(br % R), b = (int)(br / R);
    const int t = p.lo[0] + i;
    float v = __ldg(p.bf + r);
    for (int k = 0; k < ks; k++) {
      const int pp = t - (ks - 1 - k);
      if (pp >= 0) {
        int q = p.xs[(size_t)b * p.P + pp] % Q;
        if (q < 0) q += Q;
        v += __ldg(p.wf + ((size_t)k * Q + q) * R + r);
      }
    }
    x0[(size_t)br * p.nw + (t - p.base)] = v;
    if (t >= p.P - 1 - qlen) p.queues[(size_t)b * p.q_per_utt + p.qoff[0] + (size_t)(t % qlen) * R + r] = v;
  }
}

// row k of layer l's input at position t (t <= P - 2): [taps | x(t) | aux]
__device__ __forceinline__ float layer_input(const Params& p, const float* xb, int d, int k, int t, int b) {
  const int R = p.R, ks = p.ks;
  if (k < (ks - 1) * R) {
    const int j = k / R, r = k - j * R, s = (ks - 1 - j) * d;
    return t - s >= 0 ? xb[(size_t)r * p.nw + (t - s - p.base)] : 0.f;
  }
  if (k < ks * R) return xb[(size_t)(k - (ks - 1) * R) * p.nw + (t - p.base)];
  const int a = k - ks * R;
  if (a >= p.A) return 0.f;
  const int j = max(t - p.n_pad, 0);
  if (p.U > 0) {
    const int tf = min(j / p.U, p.Th - 1), jj = j % p.U;
    return fmaf(__ldg(p.h + ((size_t)b * p.A + a) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
  }
  return __ldg(p.h + ((size_t)b * p.A + a) * p.Th + min(j, p.Th - 1));
}

// x_{l+1}(t) from x_l for t in [lo[l + 1], P - 2]: one CTA per kTP positions of one utterance.  The gate runs first over
// column passes of kCB, its z kept in shared memory; the residual then reads z from there.  Thread (tx, pg) owns columns
// cb0 + tx and cb0 + tx + 64 at the positions 4 pg .. 4 pg + 3 of the tile.
__global__ void __launch_bounds__(kThreads) stream_prefill_layer_kernel(const Params p, int l, const float* xin,
                                                                        float* xout) {
  extern __shared__ __align__(16) float sm[];
  const int R = p.R;
  float* zt = sm;                          // [R][kTP]
  float* xst = zt + (size_t)R * kTP;       // [kKB][kTP]
  float* wst = xst + kKB * kTP;            // [kKB][2 kCB]
  const int tid = threadIdx.x, tx = tid & 63, pg = tid >> 6;
  const int d = p.dil[l], lo_out = p.lo[l + 1], last = p.P - 2;
  const int tiles_per = (last - lo_out + kTP) / kTP;
  const int b = blockIdx.x / tiles_per;
  const int t0 = lo_out + (blockIdx.x % tiles_per) * kTP;
  const float* xb = xin + (size_t)b * R * p.nw;
  const float* W1 = p.stream + (size_t)l * p.layer_stride;
  const float* W2 = W1 + p.off_w2res;

  // ---------------- gate ----------------
  {
    const int O = p.O1, K = p.K1;
    const int parts = parts_for(O), rpc = rows_per_chunk(O, parts);
    for (int cb0 = 0; cb0 < R; cb0 += kCB) {
      float s[2][2][4], c0[2][2][4], acc[2][2][4];   // [column i][sigmoid, tanh][position]
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int g = 0; g < 2; g++)
#pragma unroll
          for (int q = 0; q < 4; q++) s[i][g][q] = 0.f, c0[i][g][q] = 0.f;
      for (int part = 0; part < parts; part++) {
        for (int c = 0; c < 2; c++) {
          const Chain ch(K, rpc, parts, part + c * parts);
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
            for (int g = 0; g < 2; g++)
#pragma unroll
              for (int q = 0; q < 4; q++) acc[i][g][q] = 0.f;
          for (int m0 = 0; m0 < ch.n; m0 += kKB) {
            const int cnt = min(kKB, ch.n - m0);
            __syncthreads();   // the previous stage is consumed
            for (int e = tid; e < cnt * kTP; e += kThreads) {
              const int kb = e / kTP, tp = e % kTP, t = t0 + tp;
              xst[e] = t <= last ? layer_input(p, xb, d, ch.row(m0 + kb), t, b) : 0.f;
            }
            for (int e = tid; e < cnt * (2 * kCB / 4); e += kThreads) {
              const int kb = e / (2 * kCB / 4), c4 = e % (2 * kCB / 4);
              const int col = cb0 + 4 * (c4 % (kCB / 4));
              float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
              if (col < R)
                v = __ldg(reinterpret_cast<const float4*>(W1 + (size_t)ch.row(m0 + kb) * O + col +
                                                          (c4 >= kCB / 4 ? R : 0)));
              reinterpret_cast<float4*>(wst)[e] = v;
            }
            __syncthreads();
            for (int kb = 0; kb < cnt; kb++) {
              const float4 xv = *reinterpret_cast<const float4*>(xst + kb * kTP + 4 * pg);
              const float x4[4] = {xv.x, xv.y, xv.z, xv.w};
              const float* wr = wst + kb * 2 * kCB;
              const float wv[2][2] = {{wr[tx], wr[kCB + tx]}, {wr[tx + 64], wr[kCB + tx + 64]}};
#pragma unroll
              for (int i = 0; i < 2; i++)
#pragma unroll
                for (int g = 0; g < 2; g++)
#pragma unroll
                  for (int q = 0; q < 4; q++) acc[i][g][q] = fmaf(wv[i][g], x4[q], acc[i][g][q]);
            }
          }
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
            for (int g = 0; g < 2; g++)
#pragma unroll
              for (int q = 0; q < 4; q++) {
                if (c == 0) c0[i][g][q] = acc[i][g][q];
                else s[i][g][q] += c0[i][g][q] + acc[i][g][q];
              }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int col = cb0 + tx + 64 * i;
        if (col >= R) continue;
        const float ba = __ldg(p.b1 + (size_t)l * 2 * R + col), bg = __ldg(p.b1 + (size_t)l * 2 * R + R + col);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const float a = s[i][0][q] + ba;
          const float g = s[i][1][q] + bg;
          zt[(size_t)col * kTP + 4 * pg + q] = sigmoidf_(a) * tanhf(g);
        }
      }
    }
  }

  // ---------------- residual ----------------
  {
    const int O = p.Or, K = R;
    const int parts = parts_for(O), rpc = rows_per_chunk(O, parts);
    const int dn = p.dil[l + 1], qlen = (p.ks - 1) * dn;
    for (int cb0 = 0; cb0 < R; cb0 += kCB) {
      float s[2][4], c0[2][4], acc[2][4];
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int q = 0; q < 4; q++) s[i][q] = 0.f, c0[i][q] = 0.f;
      for (int part = 0; part < parts; part++) {
        for (int c = 0; c < 2; c++) {
          const Chain ch(K, rpc, parts, part + c * parts);
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[i][q] = 0.f;
          for (int m0 = 0; m0 < ch.n; m0 += kKB) {
            const int cnt = min(kKB, ch.n - m0);
            __syncthreads();   // the previous stage is consumed (first stage: z is complete)
            for (int e = tid; e < cnt * (kCB / 4); e += kThreads) {
              const int kb = e / (kCB / 4), col = cb0 + 4 * (e % (kCB / 4));
              float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
              if (col < R) v = __ldg(reinterpret_cast<const float4*>(W2 + (size_t)ch.row(m0 + kb) * O + col));
              reinterpret_cast<float4*>(wst)[e] = v;
              if (e % (kCB / 4) == 0) reinterpret_cast<int*>(xst)[kb] = ch.row(m0 + kb);
            }
            __syncthreads();
            for (int kb = 0; kb < cnt; kb++) {
              const int k = reinterpret_cast<const int*>(xst)[kb];
              const float4 zv = *reinterpret_cast<const float4*>(zt + (size_t)k * kTP + 4 * pg);
              const float z4[4] = {zv.x, zv.y, zv.z, zv.w};
              const float wv[2] = {wst[kb * kCB + tx], wst[kb * kCB + tx + 64]};
#pragma unroll
              for (int i = 0; i < 2; i++)
#pragma unroll
                for (int q = 0; q < 4; q++) acc[i][q] = fmaf(wv[i], z4[q], acc[i][q]);
            }
          }
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
            for (int q = 0; q < 4; q++) {
              if (c == 0) c0[i][q] = acc[i][q];
              else s[i][q] += c0[i][q] + acc[i][q];
            }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int col = cb0 + tx + 64 * i;
        if (col >= R) continue;
        const float bias = __ldg(p.b2 + (size_t)l * (R + p.S) + col);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int t = t0 + 4 * pg + q;
          if (t > last) continue;
          const size_t at = ((size_t)b * R + col) * p.nw + (t - p.base);
          const float v = xin[at] + (s[i][q] + bias);
          xout[at] = v;
          if (t >= p.P - 1 - qlen)
            p.queues[(size_t)b * p.q_per_utt + p.qoff[l + 1] + (size_t)(t % qlen) * R + col] = v;
        }
      }
    }
  }
}

}  // namespace dsp

int decode_stream_supported_shape(int Q, int Ap, int R, int S, int ks, int L);   // decode_stream.cu

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_decode_stream_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                      const float* wf, const float* bf, const float* stream, const float* b1,
                                      const float* b2, const int32_t* host_dilations, int L, void* queues,
                                      void* scratch, int B, int P, int n_pad, int Th, int Q, int A, int Ap, int R,
                                      int S, int ks, int U, void* stream_handle) {
  using namespace dsp;
  WNB_REQUIRE(B > 0 && P >= 1 && n_pad >= 0 && n_pad < P && Th >= 1 && Q > 0 && A > 0 && Ap >= A && R > 0 && S > 0 &&
                  ks >= 1 && U >= 0 && L >= 1,
              "decode_stream_prefill: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && stream && b1 && b2 && host_dilations && (queues || ks == 1),
              "decode_stream_prefill: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_stream_prefill: U>0 needs upsampling weight and bias");
  for (int l = 0; l < L && l < kMaxL; l++)
    WNB_REQUIRE(host_dilations[l] >= 1, "decode_stream_prefill: dilations must be >= 1");
  if (!decode_stream_supported_shape(Q, Ap, R, S, ks, L)) {
    set_error("decode_stream_prefill: shape not covered by the streaming kernel");
    return WNB_ERR_UNSUPPORTED;
  }
  Params p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf; p.stream = stream; p.b1 = b1; p.b2 = b2;
  p.queues = (float*)queues;
  p.P = P; p.n_pad = n_pad; p.Th = Th; p.Q = Q; p.A = A; p.R = R; p.S = S; p.ks = ks; p.U = U; p.L = L;
  p.O1 = (2 * R + 3) & ~3; p.Or = (R + 3) & ~3; p.K1 = ks * R + Ap;
  const int Os = (S + 3) & ~3;
  p.off_w2res = (long long)p.K1 * p.O1;
  p.layer_stride = p.off_w2res + (long long)R * p.Or + (long long)R * Os;
  long long off = 0;
  for (int l = 0; l < L; l++) {
    p.dil[l] = host_dilations[l];
    p.qoff[l] = off;
    off += (long long)(ks - 1) * host_dilations[l] * R;
  }
  p.q_per_utt = off;
  int64_t Sw[kMaxL];   // the pruned windows S_l
  wnb_decode_prefill_windows(host_dilations, L, ks, Sw);
  for (int l = 0; l < L; l++) p.lo[l] = (int)(P - 1 - Sw[l] > 0 ? P - 1 - Sw[l] : 0);
  p.base = p.lo[0];
  p.nw = P - 1 - p.lo[0];
  if (p.nw == 0) return WNB_OK;   // no queued warm-up position (P == 1, or ks == 1)
  WNB_REQUIRE(scratch, "decode_stream_prefill: null scratch");
  cudaStream_t st = (cudaStream_t)stream_handle;
  const int rows = B < kRows ? B : kRows;
  float* xa = (float*)scratch;
  float* xb = xa + (size_t)rows * R * p.nw;
  const size_t smem = ((size_t)R * kTP + kKB * kTP + kKB * 2 * kCB) * sizeof(float);
  WNB_CUDA(ensure_dynamic_smem((const void*)stream_prefill_layer_kernel, smem));
  for (int g0 = 0; g0 < B; g0 += kRows) {
    Params pg = p;
    pg.B = B - g0 < kRows ? B - g0 : kRows;
    pg.xs = xs + (size_t)g0 * P;
    pg.h = h + (size_t)g0 * A * Th;
    pg.queues = p.queues + (size_t)g0 * p.q_per_utt;
    {
      const long long total = (long long)pg.B * R * p.nw;
      const int grid = (int)(total / 256 + 1 < 65536 ? total / 256 + 1 : 65536);
      stream_prefill_front_kernel<<<grid, 256, 0, st>>>(pg, xa);
      WNB_CHECK_LAUNCH("decode_stream_prefill");
    }
    for (int l = 0; l + 1 < L; l++) {
      const int grid = pg.B * ((P - 1 - p.lo[l + 1] + kTP - 1) / kTP);
      stream_prefill_layer_kernel<<<grid, kThreads, smem, st>>>(pg, l, (l & 1) ? xb : xa, (l & 1) ? xa : xb);
      WNB_CHECK_LAUNCH("decode_stream_prefill");
    }
  }
  return WNB_OK;
}

}  // extern "C"
