// decode_prefill.cu -- the teacher-forced warm-up of decode_warp (padded positions 0 .. P - 2), computed in parallel over
// time and bit-identical to the sequential warm-up.
//
// Every x_l(t) with t < P - 1 depends only on the seed prefix xs, the aux features and the weights, so per layer all
// warm-up positions are independent, like the utterances of a batch.  What the free-running steps need from the warm-up
// is only the dilation queues: layer l's ring holds x_l(t) for t in [P - 1 - d_l, P - 2].  The kernels here write exactly
// those slots with exactly the bits decode_warp_kernel leaves there, so wnb_decode_warp_at(pos0 = P - 1) continues as if
// it had run the warm-up itself.
//
// Pruned windows (ks = 2): x_L is never queued, and x_{l+1}(t) needs x_l(t) and x_l(t - d_l), so layer l's input is
// needed on the last S_l = sum_{m >= l} d_m positions before P - 1 only (nets/wavenet.py decode_prefill_windows).  The
// work therefore does not depend on the seed length: a prompt longer than the receptive field costs what a one-sample
// seed costs.
//
// Bit identity.  decode_warp_kernel's per-element arithmetic does not depend on its launch form:
//   * a gate pre-activation is a per-lane FMA chain over K = [taps 64 | x(t) 64 | aux 32], lane a taking k = 32 j + a for
//     j = 0..4 in order from 0, followed by warp_reduce_scatter, which adds the 32 lane partials pairwise over lane bits
//     16, 8, 4, 2, 1 (float addition is commutative, so the tree is the same for every NU and W);
//   * then a = pre_s + b1, g = pre_t + b1', z = sigmoidf_(a) * tanhf(g);
//   * a residual output is the same kind of chain over z (j = 0, 1), the same tree, then (pre + b2) + x;
//   * the one form dependence: with CL = 2 the CTA owning channels 32..63 runs the residual's two K halves as j = 1, 0.
// Here one thread owns an output at two positions and walks the 32 lanes in bit-reversed order, which turns the
// butterfly into a plain pairwise sum over consecutive leaves (a 5-entry stack); the front, the aux column and the
// epilogues restate the decoder's expressions.  Plain FFMA, precise expf / tanhf, like the decoder.
#include <type_traits>

#include "common.cuh"

namespace wnb {
namespace dp {

constexpr int kR = 64, kQ = 256, kAp = 32, kK1 = 160, kG = 2 * kR, kS = 512;   // decode_warp's shape
constexpr int kMaxL = 64;
constexpr int kNT = 64;        // positions per tile
constexpr int kThreads = 256;  // 8 warps
constexpr int kSmemFloats = kK1 * kG + kR * kR + kG + kR + kK1 * kNT + kR * kNT;

struct Params {
  const int32_t* xs; const float* h; const float* up_w; const float* up_b;
  const float *wf, *bf, *w1d, *b1, *w2d, *b2;
  float* queues;
  int B, P, n_pad, Th, A, U, L, CL;
  int base, nw;              // scratch x_l: [B][64][nw], column c = position base + c
  long long q_per_utt;
  int dil[kMaxL];
  long long qoff[kMaxL];
  int lo[kMaxL];             // first position of layer l's input window: max(0, P - 1 - S_l)
};

// leaf i of the pairwise sum is lane bitrev5(i): consecutive leaves differ in lane bit 16, pairs of pairs in bit 8, ...
__host__ __device__ constexpr int bitrev5(int i) {
  return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4);
}

// x_0(t) = the front (causal) conv, for t in [lo[0], P - 2]: the decoder's prologue expression, in its order
__global__ void prefill_front_kernel(const Params p, float* x0) {
  const int n = p.P - 1 - p.lo[0];
  const long long total = (long long)p.B * kR * n;
  const int d0 = p.dil[0];
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % n);
    const long long br = e / n;
    const int r = (int)(br % kR), b = (int)(br / kR);
    const int t = p.lo[0] + i;
    float v = __ldg(p.bf + r);
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const int pp = t - (1 - k);
      if (pp >= 0) {
        int q = p.xs[(size_t)b * p.P + pp] % kQ;
        if (q < 0) q += kQ;
        v += __ldg(p.wf + ((size_t)k * kQ + q) * kR + r);
      }
    }
    x0[(size_t)br * p.nw + (t - p.base)] = v;
    if (t >= p.P - 1 - d0) p.queues[(size_t)b * p.q_per_utt + p.qoff[0] + (size_t)(t & (d0 - 1)) * kR + r] = v;
  }
}

// Pairwise sum of the 32 lane partials of NV outputs, fed one leaf at a time in bit-reversed lane order: after leaf 31,
// tot[] holds warp_reduce_scatter's totals.
template <int NV>
struct LaneTree {
  float st[5][NV];
  template <int I>
  __device__ __forceinline__ void push(float (&s)[NV], float (&tot)[NV]) {
#pragma unroll
    for (int lv = 0; lv < 5; lv++) {
      if ((I >> lv) & 1) {
#pragma unroll
        for (int e = 0; e < NV; e++) s[e] = st[lv][e] + s[e];
      } else {
#pragma unroll
        for (int e = 0; e < NV; e++) st[lv][e] = s[e];
        return;
      }
    }
#pragma unroll
    for (int e = 0; e < NV; e++) tot[e] = s[e];
  }
};

template <int I, int N>
struct Unroll {
  template <class F>
  __device__ __forceinline__ static void run(F&& f) {
    f(std::integral_constant<int, I>());
    Unroll<I + 1, N>::run(f);
  }
};
template <int N>
struct Unroll<N, N> {
  template <class F>
  __device__ __forceinline__ static void run(F&&) {}
};

// x_{l+1}(t) from x_l for t in [lo[l + 1], P - 2]: one CTA per SM keeps layer l's W1 (80 KB), W2res (16 KB) and biases in
// shared memory and walks tiles of 64 positions of one utterance.  Warp w owns gate channels 4w..4w+3 and 4(w+8)..,
// residual channels 8w..8w+7; lane holds positions lane and lane + 32 of the tile.
__global__ void __launch_bounds__(kThreads, 1) prefill_layer_kernel(const Params p, int l, const float* xin, float* xout) {
  extern __shared__ __align__(16) float sm[];
  float* w1 = sm;                    // [160 k][128 o]
  float* w2 = w1 + kK1 * kG;         // [64 k][64 c]   (residual columns of w2d)
  float* bias1 = w2 + kR * kR;       // [128]
  float* bias2 = bias1 + kG;         // [64]
  float* in = bias2 + kR;            // [160 k][64 t]: x_l(t - d) | x_l(t) | aux(t)
  float* zt = in + kK1 * kNT;        // [64 c][64 t]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  const float4* W1 = reinterpret_cast<const float4*>(p.w1d + (size_t)l * kK1 * kG);
  for (int e = tid; e < kK1 * kG / 4; e += kThreads) reinterpret_cast<float4*>(w1)[e] = __ldg(W1 + e);
  const float* W2 = p.w2d + (size_t)l * kR * (kR + kS);
  for (int e = tid; e < kR * kR / 4; e += kThreads) {
    const int k = e / (kR / 4), c4 = e % (kR / 4);
    reinterpret_cast<float4*>(w2)[e] = __ldg(reinterpret_cast<const float4*>(W2 + (size_t)k * (kR + kS)) + c4);
  }
  if (tid < kG) bias1[tid] = __ldg(p.b1 + (size_t)l * kG + tid);
  if (tid < kR) bias2[tid] = __ldg(p.b2 + (size_t)l * (kR + kS) + tid);

  const int d = p.dil[l], dn = p.dil[l + 1], lo_out = p.lo[l + 1], last = p.P - 2;
  const long long tiles_per = (last - lo_out + kNT) / kNT;
  const long long ntiles = tiles_per * p.B;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int b = (int)(tile / tiles_per);
    const int t0 = lo_out + (int)(tile % tiles_per) * kNT;
    const float* xb = xin + (size_t)b * kR * p.nw;
    __syncthreads();   // the previous tile's in / zt are consumed (first tile: the weights have landed)
    for (int e = tid; e < kK1 * kNT; e += kThreads) {
      const int k = e / kNT, t = t0 + e % kNT;
      float v = 0.f;
      if (t <= last) {
        if (k < kR) {
          if (t - d >= 0) v = xb[(size_t)k * p.nw + (t - d - p.base)];
        } else if (k < 2 * kR) {
          v = xb[(size_t)(k - kR) * p.nw + (t - p.base)];
        } else if (k - 2 * kR < p.A) {   // the decoder's aux column (fetch_aux_taps), h_frame0 = 0
          const int a = k - 2 * kR, j = max(t - p.n_pad, 0);
          if (p.U > 0) {
            const int tf = min(j / p.U, p.Th - 1), jj = j % p.U;
            v = fmaf(__ldg(p.h + ((size_t)b * p.A + a) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
          } else {
            v = __ldg(p.h + ((size_t)b * p.A + a) * p.Th + min(j, p.Th - 1));
          }
        }
      }
      in[e] = v;
    }
    __syncthreads();

    // ---- gate: outputs [sigmoid c0..c0+3 | tanh c0..c0+3] x positions (lane, lane + 32) ----
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
      const int c0 = 4 * (warp + 8 * half);
      float tot[16];
      LaneTree<16> tree;
      Unroll<0, 32>::run([&](auto I) {
        constexpr int a = bitrev5(decltype(I)::value);
        float s[16];
#pragma unroll
        for (int e = 0; e < 16; e++) s[e] = 0.f;
#pragma unroll
        for (int j = 0; j < 5; j++) {
          const int k = 32 * j + a;
          const float4 ws = *reinterpret_cast<const float4*>(w1 + k * kG + c0);
          const float4 wt = *reinterpret_cast<const float4*>(w1 + k * kG + kR + c0);
          const float wv[8] = {ws.x, ws.y, ws.z, ws.w, wt.x, wt.y, wt.z, wt.w};
#pragma unroll
          for (int u = 0; u < 2; u++) {
            const float x = in[k * kNT + lane + 32 * u];
#pragma unroll
            for (int o = 0; o < 8; o++) s[u * 8 + o] = fmaf(wv[o], x, s[u * 8 + o]);
          }
        }
        tree.template push<decltype(I)::value>(s, tot);
      });
#pragma unroll
      for (int u = 0; u < 2; u++)
#pragma unroll
        for (int cc = 0; cc < 4; cc++) {
          const float a = tot[u * 8 + cc] + bias1[c0 + cc];
          const float g = tot[u * 8 + 4 + cc] + bias1[kR + c0 + cc];
          zt[(c0 + cc) * kNT + lane + 32 * u] = sigmoidf_(a) * tanhf(g);
        }
    }
    __syncthreads();

    // ---- residual: channels 8w..8w+7 x positions (lane, lane + 32); CL = 2 runs channels 32..63 as j = 1, 0 ----
    {
      const int c0 = 8 * warp;
      const int jfirst = (p.CL == 2 && c0 >= 32) ? 1 : 0;
      float tot[16];
      LaneTree<16> tree;
      Unroll<0, 32>::run([&](auto I) {
        constexpr int a = bitrev5(decltype(I)::value);
        float s[16];
#pragma unroll
        for (int e = 0; e < 16; e++) s[e] = 0.f;
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          const int k = 32 * (jj ^ jfirst) + a;
          const float4 w0 = *reinterpret_cast<const float4*>(w2 + k * kR + c0);
          const float4 w1v = *reinterpret_cast<const float4*>(w2 + k * kR + c0 + 4);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1v.x, w1v.y, w1v.z, w1v.w};
#pragma unroll
          for (int u = 0; u < 2; u++) {
            const float z = zt[k * kNT + lane + 32 * u];
#pragma unroll
            for (int o = 0; o < 8; o++) s[u * 8 + o] = fmaf(wv[o], z, s[u * 8 + o]);
          }
        }
        tree.template push<decltype(I)::value>(s, tot);
      });
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int i = lane + 32 * u, t = t0 + i;
        if (t > last) continue;
#pragma unroll
        for (int o = 0; o < 8; o++) {
          const int c = c0 + o;
          const float v = tot[u * 8 + o] + bias2[c] + in[(kR + c) * kNT + i];
          xout[((size_t)b * kR + c) * p.nw + (t - p.base)] = v;
          if (t >= p.P - 1 - dn)
            p.queues[(size_t)b * p.q_per_utt + p.qoff[l + 1] + (size_t)(t & (dn - 1)) * kR + c] = v;
        }
      }
    }
  }
}

}  // namespace dp
}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_decode_prefill_windows(const int32_t* host_dilations, int L, int ks, int64_t* windows) {
  WNB_REQUIRE(host_dilations && windows && L >= 1 && ks >= 1, "decode_prefill_windows: bad arguments");
  for (int l = 0; l < L; l++) WNB_REQUIRE(host_dilations[l] >= 1, "decode_prefill_windows: dilations must be >= 1");
  int64_t S = 0;
  for (int l = L - 1; l >= 0; l--) {
    S += (int64_t)(ks - 1) * host_dilations[l];
    windows[l] = S;
  }
  return WNB_OK;
}

WNB_API size_t wnb_decode_prefill_workspace(int B, int P, int R, int ks, const int32_t* host_dilations, int L) {
  if (B <= 0 || P < 1 || R <= 0 || ks < 1 || L < 1 || L > dp::kMaxL) return 0;
  int64_t S[dp::kMaxL];
  if (wnb_decode_prefill_windows(host_dilations, L, ks, S) != WNB_OK) return 0;
  const int64_t nw = S[0] < P - 1 ? S[0] : P - 1;
  return 2 * (size_t)B * (size_t)R * (size_t)nw * sizeof(float);
}

WNB_API int wnb_decode_warp_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                    const float* wf, const float* bf, const float* w1d, const float* b1,
                                    const float* w2d, const float* b2, const int32_t* host_dilations, int L,
                                    void* queues, void* scratch, int B, int P, int n_pad, int Th, int A, int U, int CL,
                                    void* stream_handle) {
  using namespace dp;
  WNB_REQUIRE(B > 0 && P >= 1 && n_pad >= 0 && n_pad < P && Th >= 1 && A > 0 && A <= kAp && U >= 0 && L >= 1 &&
                  L <= kMaxL && (CL == 1 || CL == 2),
              "decode_warp_prefill: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && w1d && b1 && w2d && b2 && host_dilations && queues,
              "decode_warp_prefill: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_warp_prefill: U>0 needs upsampling weight and bias");
  Params p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf; p.w1d = w1d; p.b1 = b1; p.w2d = w2d;
  p.b2 = b2; p.queues = (float*)queues;
  p.B = B; p.P = P; p.n_pad = n_pad; p.Th = Th; p.A = A; p.U = U; p.L = L; p.CL = CL;
  long long off = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1 && (host_dilations[l] & (host_dilations[l] - 1)) == 0,
                "decode_warp_prefill: dilations must be powers of two");
    p.dil[l] = host_dilations[l];
    p.qoff[l] = off;
    off += (long long)host_dilations[l] * kR;
  }
  p.q_per_utt = off;
  int64_t S[kMaxL];   // the pruned windows S_l (ks = 2)
  wnb_decode_prefill_windows(host_dilations, L, 2, S);
  for (int l = 0; l < L; l++) p.lo[l] = (int)(P - 1 - S[l] > 0 ? P - 1 - S[l] : 0);
  p.base = p.lo[0];
  p.nw = P - 1 - p.lo[0];
  WNB_REQUIRE(scratch || p.nw == 0, "decode_warp_prefill: null scratch");
  if (p.nw == 0) return WNB_OK;   // P == 1: no warm-up position
  cudaStream_t st = (cudaStream_t)stream_handle;
  float* xa = (float*)scratch;
  float* xb = xa + (size_t)B * kR * p.nw;
  {
    const long long total = (long long)B * kR * p.nw;
    const int grid = (int)(total / 256 + 1 < 65536 ? total / 256 + 1 : 65536);
    prefill_front_kernel<<<grid, 256, 0, st>>>(p, xa);
    WNB_CHECK_LAUNCH("decode_warp_prefill");
  }
  const size_t smem = (size_t)kSmemFloats * sizeof(float);
  WNB_CUDA(ensure_dynamic_smem((const void*)prefill_layer_kernel, smem));
  for (int l = 0; l + 1 < L; l++) {
    const long long ntiles = (long long)B * ((P - 1 - p.lo[l + 1] + kNT - 1) / kNT);
    const int grid = (int)(ntiles < device_sms() ? ntiles : device_sms());
    prefill_layer_kernel<<<grid, kThreads, smem, st>>>(p, l, (l & 1) ? xb : xa, (l & 1) ? xa : xb);
    WNB_CHECK_LAUNCH("decode_warp_prefill");
  }
  return WNB_OK;
}

}  // extern "C"
