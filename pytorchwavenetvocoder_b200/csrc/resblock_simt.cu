// resblock_simt.cu -- WNB_MATH_FP32 kernels for the residual stack and the post network.
//
//   resblock_fwd_simt_kernel : ONE launch per residual block (wavenet.py:525-536): dilated causal conv
//                              (both branches) + aux 1x1 + sigmoid*tanh gate + res/skip 1x1 + residual
//                              add + running skip accumulation.  The gate tile never leaves shared memory.
//   resblock_bwd_gate_kernel : recomputes the gate from (xin, haux), forms dz = W2^T [dout|dskip] and
//                              writes z and dpre = [dz*th*sg*(1-sg) | dz*sg*(1-th^2)].
//   gemm_nt_kernel           : C[t][m] = sum_seg sum_k A_seg[m][k] * B_seg[t+shift][k] (+bias, +add, relu,
//                              mask, accumulate): used for the data gradients and the post network.
//   gemm_tn_kernel           : weight gradients  dW[m][n] += sum_t A[t][m] * B[t+shift][n], split over (batch, time
//                              range); colsum_kernel: bias gradients, split over row ranges.  Each CTA writes its
//                              partial sum to its own slot of a per-stream scratch and slot_reduce_kernel adds the
//                              slots in slot order (no atomics: the gradients do not depend on scheduling).
//
// All activations are channels-last (B,T,C).  Everything here is fp32 FFMA: this is the parity path and
// the fallback for shapes the tensor-core paths do not cover.
#include <stdlib.h>

#include <initializer_list>
#include <utility>

#include "gemm_simt.cuh"
#include "tc_host.h"

namespace wnb {

// ------------------------------------------------------------------------------------------------
// fused residual block forward
// ------------------------------------------------------------------------------------------------
struct FwdParams {
  const float* xin; const float* haux; const float* w1; const float* b1; const float* w2; const float* b2;
  float* xout; float* skip; float* zsave;
  int B, T, R, S, Ap, ks, d, skip_init;
};

__global__ void __launch_bounds__(kThreads) resblock_fwd_simt_kernel(FwdParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<8>& sm = *reinterpret_cast<TileSmem<8>*>(smem_raw);
  float* zs = reinterpret_cast<float*>(smem_raw + sizeof(TileSmem<8>));  // [R][kBsLd], k-major gate tile

  const int b = blockIdx.y, t0 = blockIdx.x * kBN;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int R = p.R, S = p.S, Ap = p.Ap, ks = p.ks, d = p.d, T = p.T;
  const int K1 = ks * R + Ap;
  const float* xin_b = p.xin + (size_t)b * T * R;
  const float* haux_b = p.haux + (size_t)b * T * Ap;

  // ---- phase 1: pre-activations, 64 gate channels (128 interleaved W1 rows) at a time ----
  for (int gc = 0; gc < R; gc += 64) {
    float acc[8][kTN];
    zero_acc<8>(acc);
    auto fa = [&](int m, int k) -> float {
      const int c = gc + (m >> 1);
      if (c >= R) return 0.f;
      const int row = (m & 1) ? R + c : c;
      return __ldg(p.w1 + (size_t)row * K1 + k);
    };
    auto fb = [&](int n, int k) -> float {
      const int t = t0 + n;
      if (t >= T) return 0.f;
      if (k < ks * R) {
        const int j = k / R, c = k - j * R;
        const int tt = t - (ks - 1 - j) * d;
        return tt >= 0 ? __ldg(xin_b + (size_t)tt * R + c) : 0.f;
      }
      return __ldg(haux_b + (size_t)t * Ap + (k - ks * R));
    };
    tile_mainloop<8, true, true>(acc, fa, fb, K1, sm);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int c = gc + ty * 4 + i;
      if (c < R) {
        const float bs = __ldg(p.b1 + c), bt = __ldg(p.b1 + R + c);
#pragma unroll
        for (int j = 0; j < kTN; j++)
          zs[c * kBsLd + tx * 4 + j] = sigmoidf_(acc[2 * i][j] + bs) * tanhf(acc[2 * i + 1][j] + bt);
      }
    }
  }
  __syncthreads();

  if (p.zsave) {
    float* zb = p.zsave + (size_t)b * T * R;
    for (int e = tid; e < kBN * R; e += kThreads) {
      const int c = e % R, n = e / R;
      if (t0 + n < T) zb[(size_t)(t0 + n) * R + c] = zs[c * kBsLd + n];
    }
  }

  // ---- phase 2: [res | skip] 1x1 on the gate tile, 128 output rows at a time ----
  const int row_begin = p.xout ? 0 : R;  // last layer: residual output is discarded
  const int M2 = R + S;
  float* xout_b = p.xout ? p.xout + (size_t)b * T * R : nullptr;
  float* skip_b = p.skip + (size_t)b * T * S;
  for (int r0 = row_begin; r0 < M2; r0 += 128) {
    float acc[8][kTN];
    zero_acc<8>(acc);
    auto fa = [&](int m, int k) -> float {
      const int row = r0 + m;
      return row < M2 ? __ldg(p.w2 + (size_t)row * R + k) : 0.f;
    };
    auto fb = [&](int n, int k) -> float { return zs[k * kBsLd + n]; };
    tile_mainloop<8, true, false>(acc, fa, fb, R, sm);
#pragma unroll
    for (int j = 0; j < kTN; j++) {
      const int t = t0 + tx * 4 + j;
      if (t >= T) continue;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int row = r0 + ty * 8 + i;
        if (row >= M2) continue;
        const float v = acc[i][j] + __ldg(p.b2 + row);
        if (row < R) {
          xout_b[(size_t)t * R + row] = v + __ldg(xin_b + (size_t)t * R + row);
        } else {
          float* dst = skip_b + (size_t)t * S + (row - R);
          *dst = p.skip_init ? v : (*dst + v);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward, gate part: recompute sg/th, dz, write z and dpre
// ------------------------------------------------------------------------------------------------
struct BwdGateParams {
  const float* xin; const float* haux; const float* dout; const float* dskip;
  const float* w1; const float* b1; const float* w2t;  // w2t (R, R+S): [c][o]
  float* z; float* dpre;                               // (B,T,R), (B,T,2R)
  int B, T, R, S, Ap, ks, d;
};

__global__ void __launch_bounds__(kThreads) resblock_bwd_gate_kernel(BwdGateParams p) {
  __shared__ TileSmem<8> sm8;
  TileSmem<4>& sm4 = *reinterpret_cast<TileSmem<4>*>(&sm8);
  const int b = blockIdx.y, t0 = blockIdx.x * kBN, gc = blockIdx.z * 64;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int R = p.R, S = p.S, Ap = p.Ap, ks = p.ks, d = p.d, T = p.T;
  const int K1 = ks * R + Ap, M2 = R + S;
  const float* xin_b = p.xin + (size_t)b * T * R;
  const float* haux_b = p.haux + (size_t)b * T * Ap;
  const float* dout_b = p.dout ? p.dout + (size_t)b * T * R : nullptr;
  const float* dskip_b = p.dskip + (size_t)b * T * S;

  float sg[4][kTN], th[4][kTN];
  {
    float acc[8][kTN];
    zero_acc<8>(acc);
    auto fa = [&](int m, int k) -> float {
      const int c = gc + (m >> 1);
      if (c >= R) return 0.f;
      const int row = (m & 1) ? R + c : c;
      return __ldg(p.w1 + (size_t)row * K1 + k);
    };
    auto fb = [&](int n, int k) -> float {
      const int t = t0 + n;
      if (t >= T) return 0.f;
      if (k < ks * R) {
        const int j = k / R, c = k - j * R;
        const int tt = t - (ks - 1 - j) * d;
        return tt >= 0 ? __ldg(xin_b + (size_t)tt * R + c) : 0.f;
      }
      return __ldg(haux_b + (size_t)t * Ap + (k - ks * R));
    };
    tile_mainloop<8, true, true>(acc, fa, fb, K1, sm8);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int c = gc + ty * 4 + i;
      const float bs = c < R ? __ldg(p.b1 + c) : 0.f, bt = c < R ? __ldg(p.b1 + R + c) : 0.f;
#pragma unroll
      for (int j = 0; j < kTN; j++) {
        sg[i][j] = sigmoidf_(acc[2 * i][j] + bs);
        th[i][j] = tanhf(acc[2 * i + 1][j] + bt);
      }
    }
  }
  float dz[4][kTN];
  zero_acc<4>(dz);
  {
    const int kofs = dout_b ? 0 : R;  // last layer: no dout, only the skip rows of W2 contribute
    auto fa = [&](int m, int k) -> float {
      const int c = gc + m;
      return c < R ? __ldg(p.w2t + (size_t)c * M2 + kofs + k) : 0.f;
    };
    auto fb = [&](int n, int k) -> float {
      const int t = t0 + n;
      if (t >= T) return 0.f;
      const int kk = kofs + k;
      return kk < R ? __ldg(dout_b + (size_t)t * R + kk) : __ldg(dskip_b + (size_t)t * S + (kk - R));
    };
    tile_mainloop<4, true, true>(dz, fa, fb, M2 - kofs, sm4);
  }
  float* z_b = p.z + (size_t)b * T * R;
  float* dpre_b = p.dpre + (size_t)b * T * 2 * R;
#pragma unroll
  for (int j = 0; j < kTN; j++) {
    const int t = t0 + tx * 4 + j;
    if (t >= T) continue;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int c = gc + ty * 4 + i;
      if (c >= R) continue;
      const float s_ = sg[i][j], h_ = th[i][j], g = dz[i][j];
      z_b[(size_t)t * R + c] = s_ * h_;
      dpre_b[(size_t)t * 2 * R + c] = g * h_ * s_ * (1.f - s_);
      dpre_b[(size_t)t * 2 * R + R + c] = g * s_ * (1.f - h_ * h_);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// generic NT GEMM over channels-last activations
// ------------------------------------------------------------------------------------------------
struct NtSeg {
  const float* a; int lda;   // A rows: a + m*lda + k
  const float* b; int ldb;   // B rows: b + (batch*T + t + shift)*ldb + k, valid iff 0 <= t+shift < T
  int shift; int K;
};
struct NtParams {
  NtSeg seg[4]; int nseg;
  int M, T, B;
  const float* bias;               // (M) or null
  float* c; int ldc;               // c[(batch*T+t)*ldc + m]
  const float* add; int ldadd;     // optional residual add (same indexing), null = none
  const float* mask; int ldmask;   // optional: multiply by (mask > 0)
  int relu_b, relu_out, accumulate;
};

__global__ void __launch_bounds__(kThreads) gemm_nt_kernel(NtParams p) {
  __shared__ TileSmem<8> sm;
  const int bidx = blockIdx.z, t0 = blockIdx.x * kBN, m0 = blockIdx.y * 128;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int T = p.T;
  float acc[8][kTN];
  zero_acc<8>(acc);
  for (int s = 0; s < p.nseg; s++) {
    const NtSeg sg = p.seg[s];
    const float* bb = sg.b + (size_t)bidx * T * sg.ldb;
    const int relu_b = p.relu_b;
    auto fa = [&](int m, int k) -> float {
      return (m0 + m < p.M) ? __ldg(sg.a + (size_t)(m0 + m) * sg.lda + k) : 0.f;
    };
    auto fb = [&](int n, int k) -> float {
      const int t = t0 + n + sg.shift;
      if (t0 + n >= T || t < 0 || t >= T) return 0.f;
      const float v = __ldg(bb + (size_t)t * sg.ldb + k);
      return relu_b ? fmaxf(v, 0.f) : v;
    };
    tile_mainloop<8, true, true>(acc, fa, fb, sg.K, sm);
  }
#pragma unroll
  for (int j = 0; j < kTN; j++) {
    const int t = t0 + tx * 4 + j;
    if (t >= T) continue;
    const size_t row = (size_t)bidx * T + t;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int m = m0 + ty * 8 + i;
      if (m >= p.M) continue;
      float v = acc[i][j];
      if (p.bias) v += __ldg(p.bias + m);
      if (p.add) v += __ldg(p.add + row * p.ldadd + m);
      if (p.relu_out) v = fmaxf(v, 0.f);
      if (p.mask) v = (__ldg(p.mask + row * p.ldmask + m) > 0.f) ? v : 0.f;
      float* dst = p.c + row * p.ldc + m;
      *dst = p.accumulate ? (*dst + v) : v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// weight gradient: C[m][coff+n] += sum_{b, t in split} A[b][t][m] * Bm[b][t+shift][n]
// ------------------------------------------------------------------------------------------------
struct TnParams {
  const float* a; int lda; int M;
  const float* b; int ldb; int N; int shift; int relu_b;
  float* c; int ldc; int coff;
  int T, B, tchunk;
  float* part;   // (B * nsplit, M, N) slot per (batch, time range), set by launch_tn; null: one slot, += straight into c
};

__global__ void __launch_bounds__(kThreads) gemm_tn_kernel(TnParams p) {
  __shared__ TileSmem<8> sm;
  const int m0 = blockIdx.x * 128, n0 = blockIdx.y * kBN;
  const int nsplit = (p.T + p.tchunk - 1) / p.tchunk;
  const int bidx = blockIdx.z / nsplit, tb = (blockIdx.z % nsplit) * p.tchunk;
  const int tlen = min(p.tchunk, p.T - tb);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const float* ab = p.a + ((size_t)bidx * p.T + tb) * p.lda;
  const float* bb = p.b + (size_t)bidx * p.T * p.ldb;
  float acc[8][kTN];
  zero_acc<8>(acc);
  auto fa = [&](int m, int k) -> float { return (m0 + m < p.M) ? __ldg(ab + (size_t)k * p.lda + m0 + m) : 0.f; };
  auto fb = [&](int n, int k) -> float {
    const int t = tb + k + p.shift;
    if (n0 + n >= p.N || t < 0 || t >= p.T) return 0.f;
    const float v = __ldg(bb + (size_t)t * p.ldb + n0 + n);
    return p.relu_b ? fmaxf(v, 0.f) : v;
  };
  tile_mainloop<8, false, false>(acc, fa, fb, tlen, sm);
  float* slot = p.part ? p.part + (size_t)blockIdx.z * p.M * p.N : nullptr;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int m = m0 + ty * 8 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < kTN; j++) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      if (slot) slot[(size_t)m * p.N + n] = acc[i][j];
      else p.c[(size_t)m * p.ldc + p.coff + n] += acc[i][j];
    }
  }
}

// sum over rows of a[row][m] (rows = B*T) in ranges of rows_per_block: block i writes part[i][m], or adds into out[m]
// when part is null (a single block)
__global__ void colsum_kernel(const float* __restrict__ a, int lda, int M, int64_t rows, int rows_per_block,
                              float* __restrict__ part, float* __restrict__ out) {
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t r1 = min(r0 + rows_per_block, rows);
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float s = 0.f;
    for (int64_t r = r0; r < r1; r++) s += a[r * lda + m];
    if (part) part[(size_t)blockIdx.x * M + m] = s;
    else out[m] += s;
  }
}

// c[m][coff + n] += part[0][m][n] + part[1][m][n] + ... + part[nslots-1][m][n], added in slot order
__global__ void slot_reduce_kernel(const float* __restrict__ part, int nslots, int M, int N, float* __restrict__ c, int ldc,
                                   int coff) {
  const int64_t mn = (int64_t)M * N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < mn; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < nslots; z++) s += part[z * mn + i];
    const int m = (int)(i / N), n = (int)(i - (int64_t)m * N);
    c[(size_t)m * ldc + coff + n] += s;
  }
}

static int launch_nt(const NtParams& p, cudaStream_t st) {
  dim3 grid(cdiv(p.T, kBN), cdiv(p.M, 128), p.B);
  gemm_nt_kernel<<<grid, kThreads, 0, st>>>(p);
  WNB_CHECK_LAUNCH("gemm_nt");
  return WNB_OK;
}

// the per-stream scratch the partial sums of one launch go to (the launches of a stream run one after the other)
static float* simt_slots(cudaStream_t st, int64_t floats) {
  float* part = static_cast<float*>(scratch_buffer(st, SCRATCH_SIMT, (size_t)floats * sizeof(float)));
  if (!part) set_error("fp32 gradients: cannot allocate the partial-sum scratch (%lld floats)", (long long)floats);
  return part;
}

static int launch_slot_reduce(const float* part, int nslots, int M, int N, float* c, int ldc, int coff, cudaStream_t st) {
  const int64_t mn = (int64_t)M * N;
  const int grid = (int)(cdiv64(mn, 256) < device_sms() * 8 ? cdiv64(mn, 256) : device_sms() * 8);
  slot_reduce_kernel<<<grid, 256, 0, st>>>(part, nslots, M, N, c, ldc, coff);
  WNB_CHECK_LAUNCH("slot_reduce");
  return WNB_OK;
}

static int launch_tn(TnParams p, cudaStream_t st) {
  const int nsplit = cdiv(p.T, p.tchunk), nslots = p.B * nsplit;
  p.part = nullptr;
  if (nslots > 1 && !(p.part = simt_slots(st, (int64_t)nslots * p.M * p.N))) return WNB_ERR_CUDA;
  dim3 grid(cdiv(p.M, 128), cdiv(p.N, kBN), nslots);
  gemm_tn_kernel<<<grid, kThreads, 0, st>>>(p);
  WNB_CHECK_LAUNCH("gemm_tn");
  return p.part ? launch_slot_reduce(p.part, nslots, p.M, p.N, p.c, p.ldc, p.coff, st) : WNB_OK;
}

static int launch_colsum(const float* a, int lda, int M, int64_t rows, float* out, cudaStream_t st) {
  const int rpb = 512;
  const int threads = M >= 256 ? 256 : ((M + 31) / 32) * 32;
  const int nblocks = (int)cdiv64(rows, rpb);
  float* part = nullptr;
  if (nblocks > 1 && !(part = simt_slots(st, (int64_t)nblocks * M))) return WNB_ERR_CUDA;
  colsum_kernel<<<nblocks, threads, 0, st>>>(a, lda, M, rows, rpb, part, out);
  WNB_CHECK_LAUNCH("colsum");
  return part ? launch_slot_reduce(part, nblocks, 1, M, out, 0, 0, st) : WNB_OK;
}

static int pick_tchunk(int B, int T, int tiles) {
  // aim for ~2 waves of CTAs over the SMs; chunks are multiples of 16 time steps
  int64_t want = (int64_t)device_sms() * 2;
  int nsplit = (int)((want + (int64_t)tiles * B - 1) / ((int64_t)tiles * B));
  if (nsplit < 1) nsplit = 1;
  int chunk = (T + nsplit - 1) / nsplit;
  chunk = ((chunk + 15) / 16) * 16;
  if (chunk < 64) chunk = 64;
  return chunk;
}

// N == 512 GEMMs of the post network as two explicit 256-column blocks (WNB_POST_SPLIT=0: one N = 512 call, which
// gemm_nt_tc splits the same way)
static bool post_split(int S) {
  static int on = -1;
  if (on < 0) { const char* e = getenv("WNB_POST_SPLIT"); on = (e && e[0] == '0') ? 0 : 1; }
  return on == 1 && S == 512;
}

static bool nt_tc_n_ok(int N) { return N % 32 == 0 && N >= 32 && (N <= 256 || N == 512); }

__global__ void relu_inplace_kernel(float4* __restrict__ x, int64_t n4) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = x[i];
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    x[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// bf16 operand path (WNB_MATH_BF16): the weights an entry call multiplies with, rounded to bf16
// ------------------------------------------------------------------------------------------------
// The ABI keeps fp32 master weights.  A bf16 entry call first rounds the matrices it uses (nearest even) into the
// per-stream SCRATCH_BF16 buffer with ONE launch; every copy starts on a 256-byte boundary.  The copies are rewritten by
// the next bf16 call on the same stream, which is ordered after every kernel of this one.
constexpr int kMaxBf16Mats = 4;
struct Bf16Job { const float* src[kMaxBf16Mats]; __nv_bfloat16* dst[kMaxBf16Mats]; int64_t n[kMaxBf16Mats]; int count; };

__global__ void to_bf16_kernel(const __grid_constant__ Bf16Job j) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int m = 0; m < j.count; m++)
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < j.n[m]; i += stride)
      j.dst[m][i] = __float2bfloat16_rn(j.src[m][i]);
}

// fp32 matrix -> its bf16 copy, looked up by the fp32 pointer the GEMM segments carry
struct Bf16Weights {
  const float* src[kMaxBf16Mats] = {};
  const __nv_bfloat16* dst[kMaxBf16Mats] = {};
  int count = 0;
  const __nv_bfloat16* of(const float* w) const {
    for (int i = 0; i < count; i++)
      if (src[i] == w) return dst[i];
    return nullptr;
  }
  // the segments' bf16 weights (no-op for a null table: the tf32 path)
  static void apply(const Bf16Weights* bw, NtTcSeg* segs, int n) {
    if (bw)
      for (int i = 0; i < n; i++) segs[i].wb = bw->of(segs[i].w);
  }
};

// mats: (fp32 matrix, element count)
static int to_bf16_weights(Bf16Weights& bw, std::initializer_list<std::pair<const float*, int64_t>> mats, cudaStream_t st) {
  Bf16Job j{};
  size_t off[kMaxBf16Mats], bytes = 0;
  for (const auto& m : mats) {
    off[j.count] = bytes;
    bytes += ((size_t)m.second * sizeof(__nv_bfloat16) + 255) & ~(size_t)255;
    j.src[j.count] = m.first;
    j.n[j.count] = m.second;
    j.count++;
  }
  unsigned char* base = static_cast<unsigned char*>(scratch_buffer(st, SCRATCH_BF16, bytes));
  if (!base) { set_error("bf16: cannot allocate the weight scratch"); return WNB_ERR_CUDA; }
  bw.count = j.count;
  for (int i = 0; i < j.count; i++) {
    j.dst[i] = reinterpret_cast<__nv_bfloat16*>(base + off[i]);
    bw.src[i] = j.src[i];
    bw.dst[i] = j.dst[i];
  }
  to_bf16_kernel<<<device_sms() * 4, 256, 0, st>>>(j);
  WNB_CHECK_LAUNCH("to_bf16");
  return WNB_OK;
}

// weight gradient C (M x N) += A^T B for arbitrary M (blocks of 128 rows, TMA zero fill past the tensor) and
// N (chunks of <= 7 groups of 32), optional bias gradient db (M) = column sums of A
static int wgrad_tc_full(const float* a, int CA, int M, const float* b, int CB, int N, float* c, int ldc, float* db,
                         int B, int T, cudaStream_t st) {
  int rc;
  for (int m0 = 0; m0 < M; m0 += 128) {
    const int m_valid = (M - m0) < 128 ? (M - m0) : 128;
    const WgOperand ao[1] = {{a, CA, m0, 4, 0}};
    for (int n0 = 0; n0 < N; n0 += 224) {
      const int groups = ((N - n0) < 224 ? (N - n0) : 224) / 32;
      const WgOperand bo[1] = {{b, CB, n0, groups, 0}};
      if ((rc = wgrad_tc(ao, 1, bo, 1, c + (size_t)m0 * ldc + n0, ldc, m_valid, (n0 == 0 && db) ? db + m0 : nullptr, B, T,
                         st)) != WNB_OK)
        return rc;
    }
  }
  return WNB_OK;
}

// C (M x N, ldc) += A^T B, db (M) += colsum A, with A = channels [0, M) of a (CA), B = channels [0, N) of b (CB):
// up to 4 M-blocks per launch and the N axis split into column groups handled by
// different CTAs (WgOpts::n_split), so a 512 x 512 gradient is ONE launch that streams A and B once from HBM.
static int wgrad_tc_split(const float* a, int CA, int M, const float* b, int CB, int N, float* c, int ldc, float* db,
                          int B, int T, cudaStream_t st) {
  int rc;
  for (int m0 = 0; m0 < M; m0 += 512) {
    WgBlock blk[4];
    int nblk = 0;
    for (int m = m0; m < M && nblk < 4; m += 128, nblk++) {
      blk[nblk].nops = 1;
      blk[nblk].ops[0] = WgOperand{a, CA, m, 4, 0};
      blk[nblk].c = c + (size_t)m * ldc;
      blk[nblk].m_valid = (M - m) < 128 ? (M - m) : 128;
      blk[nblk].db = db ? db + m : nullptr;
    }
    const int groups = N / 32, budget = 512 / nblk / 32 - (db ? 1 : 0);
    int nB = 0;
    for (int g = budget < 7 ? budget : 7; g >= 1 && !nB; g--)
      if (groups % g == 0) nB = g;
    if (!nB || groups / nB > 128) return wgrad_tc_full(a, CA, M, b, CB, N, c, ldc, db, B, T, st);
    const WgOperand bo[1] = {{b, CB, 0, nB, 0}};
    const WgOpts o{groups / nB};
    if ((rc = wgrad_tc_blocks(blk, nblk, bo, 1, ldc, B, T, st, &o)) != WNB_OK) return rc;
  }
  return WNB_OK;
}

// Weight gradient with A = the channel concatenation [a0 (C0) | a1 (C1)] (a1 may be null), M = rows used,
// B = channels [0, N) of tensor b (CB channels) read at time t + shift:  C (M x N, ldc) += A^T B, db (M) += colsum A.
// M-blocks of 128 rows are batched per launch (up to 5); N goes in chunks of <= 224 columns.
static int wgrad_tc_concat(const float* a0, int C0, const float* a1, int C1, int M, const float* b, int CB, int N,
                           int shift, float* c, int ldc, float* db, int B, int T, cudaStream_t st, bool bf16 = false) {
  // The N axis is split into column groups handled by different CTAs of ONE launch (WgOpts::n_split, as wgrad_tc_split
  // does): every launch then streams its M-blocks of A once and B once, with the B columns shared through L2 -- instead
  // of one launch per (<= 224-column chunk) x (M-block pair) that re-reads the A tensor for every chunk (the recipes'
  // 512 / 256 shape spent 41 % of its step in 897 such launches).
  int rc;
  const int groups = N / 32;
  if (N % 32 != 0 || groups < 1) { set_error("wgrad_tc_concat: N must be a multiple of 32"); return WNB_ERR_INVALID; }
  // column groups of <= 128 columns per CTA (largest divisor of N/32 up to 4)
  int nB = 1;
  for (int g = 4; g >= 1; g--)
    if (groups % g == 0 && groups / g <= 128) { nB = g; break; }
  int per_launch = 5;
  {  // same number of launches, evenly filled (4 M-blocks: 2 + 2 rather than 3 + 1)
    const int mblocks = (M + 127) / 128, launches = (mblocks + per_launch - 1) / per_launch;
    per_launch = (mblocks + launches - 1) / launches;
  }
  const int n_split = groups / nB;
  const WgOperand bo[1] = {{b, CB, 0, nB, shift}};
  WgOpts o{n_split};
  o.bf16 = bf16 ? 1 : 0;
  WgBlock blk[5];
  int nblk = 0;
  for (int m0 = 0; m0 < M; m0 += 128) {
    WgBlock& bk = blk[nblk];
    bk.m_valid = (M - m0) < 128 ? (M - m0) : 128;
    bk.c = c + (size_t)m0 * ldc;
    bk.db = db ? db + m0 : nullptr;
    // rows m0..m0+127 of the concatenation, in groups of 32 channels
    if (m0 + 128 <= C0 || !a1) {
      bk.nops = 1;
      bk.ops[0] = WgOperand{a0, C0, m0, 4, 0};            // (groups past C0 are TMA zero fill)
    } else if (m0 >= C0) {
      bk.nops = 1;
      bk.ops[0] = WgOperand{a1, C1, m0 - C0, 4, 0};
    } else {
      const int g0 = (C0 - m0) / 32;                       // groups still inside a0
      bk.nops = 2;
      bk.ops[0] = WgOperand{a0, C0, m0, g0, 0};
      bk.ops[1] = WgOperand{a1, C1, 0, 4 - g0, 0};
    }
    if (++nblk == per_launch || m0 + 128 >= M) {
      if ((rc = wgrad_tc_blocks(blk, nblk, bo, 1, ldc, B, T, st, (n_split > 1 || bf16) ? &o : nullptr)) != WNB_OK)
        return rc;
      nblk = 0;
    }
  }
  return WNB_OK;
}

// shapes the composed tensor-core path covers (generic wgmma GEMMs + gate epilogues per 64-channel chunk)
static bool composed_tc_supported(int R, int S, int Ap, int ks) {
  return R % 64 == 0 && nt_tc_n_ok(R) && nt_tc_n_ok(S) && Ap % 32 == 0 && Ap <= 256 && ks >= 1 && ks <= 3;
}

// gate channels per composed gate GEMM, and the column blocking / two-time-tile option of the plain composed GEMMs
static int composed_gc(int R) { return (R % 128 == 0) ? 128 : 64; }
static NtTcOpts plain_opts(int N) {
  NtTcOpts o{1};
  if (N > 256 && N % 256 == 0) o.n_blocks = N / 256;
  return o;
}

// Forward of one residual block for shapes outside the fused kernel: R/64 gate GEMMs (N = 128: 64 sigmoid + 64
// tanh rows of W1, K = ks*R + Ap streamed) with the gate epilogue writing z, then the res GEMM (+bias, +x) and the
// skip GEMM (+bias, store or reduce-add).  z (B,T,R) goes through p.zsave.  bw: bf16 copies of w1 / w2 (bf16 operand
// path), or null (tf32).
static int resblock_fwd_composed(const FwdParams& p, cudaStream_t st, const Bf16Weights* bw = nullptr) {
  const int R = p.R, S = p.S, Ap = p.Ap, ks = p.ks, K1 = ks * R + Ap;
  NtTcSeg segs[4];
  int ns = 0, rc;
  for (int j = 0; j < ks; j++) segs[ns++] = NtTcSeg{p.xin, R, -(ks - 1 - j) * p.d, R, p.w1, 2 * R, K1, j * R, 0};
  segs[ns++] = NtTcSeg{p.haux, Ap, 0, Ap, p.w1, 2 * R, K1, ks * R, 0};
  Bf16Weights::apply(bw, segs, ns);
  // 128 gate channels (N = 256) and two time tiles per CTA tile when R allows: the activation tile [x taps | aux] is
  // re-read R/128 instead of R/64 times and every weight chunk serves 256 rows (these GEMMs are L2 -> SM bound)
  const int GC = composed_gc(R);
    for (int c0 = 0; c0 < R; c0 += GC) {
    const NtTcGate g{1, c0, R, p.b1 + c0, p.b1 + R + c0, nullptr, nullptr};
    if ((rc = gemm_nt_tc(segs, ns, 2 * GC, p.zsave, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, p.B, p.T, st, nullptr, nullptr,
                         nullptr, 0, 0, &g)) != WNB_OK)
      return rc;
  }
  if (p.xout) {
    NtTcSeg sr[1] = {{p.zsave, R, 0, R, p.w2, R + S, R, 0, 0}};
    Bf16Weights::apply(bw, sr, 1);
    const NtTcOpts o = plain_opts(R);
    if ((rc = gemm_nt_tc(sr, 1, R / o.n_blocks, p.xout, R, p.b2, nullptr, 0, p.xin, R, 0, 0, p.B, p.T, st, nullptr, nullptr,
                         nullptr, 0, 0, nullptr, &o)) != WNB_OK)
      return rc;
  }
  NtTcSeg ss[1] = {{p.zsave, R, 0, R, p.w2, R + S, R, 0, R}};
  Bf16Weights::apply(bw, ss, 1);
  const NtTcOpts o = plain_opts(S);
  return gemm_nt_tc(ss, 1, S / o.n_blocks, p.skip, S, p.b2 + R, nullptr, 0, nullptr, 0, 0, p.skip_init ? 0 : 1, p.B, p.T, st,
                    nullptr, nullptr, nullptr, 0, 0, nullptr, &o);
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_resblock_fwd(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2,
                     const float* b2, float* xout, float* skip, float* zsave, int B, int T, int R, int S, int Ap,
                     int ks, int dilation, int skip_init, int math_mode, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && R > 0 && S > 0 && Ap > 0 && ks >= 1 && dilation >= 1, "resblock_fwd: bad shape");
  WNB_REQUIRE(xin && haux && w1 && b1 && w2 && b2 && skip, "resblock_fwd: null pointer");
  FwdParams p{xin, haux, w1, b1, w2, b2, xout, skip, zsave, B, T, R, S, Ap, ks, dilation, skip_init};
  if (math_mode == WNB_MATH_BF16) {
    // bf16 operands: the composed path for every shape it covers (the fused kernel is tf32 only)
    WNB_REQUIRE(composed_tc_supported(R, S, Ap, ks), "resblock_fwd: shape R=%d S=%d Ap=%d ks=%d not supported by the "
                "bf16 tensor-core path (use WNB_MATH_TF32 or WNB_MATH_FP32)", R, S, Ap, ks);
    cudaStream_t st = (cudaStream_t)stream;
    Bf16Weights bw;
    int rc = to_bf16_weights(bw, {{w1, (int64_t)2 * R * (ks * R + Ap)}, {w2, (int64_t)(R + S) * R}}, st);
    if (rc != WNB_OK) return rc;
    if (zsave) return resblock_fwd_composed(p, st, &bw);
    float* z = nullptr;
    WNB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&z), (size_t)B * T * R * sizeof(float), st));
    p.zsave = z;
    rc = resblock_fwd_composed(p, st, &bw);
    WNB_CUDA(cudaFreeAsync(z, st));
    return rc;
  }
  if (math_mode == WNB_MATH_TF32) {
    if (resblock_fwd_skip_supported(R, S, Ap, ks)) {
      WNB_REQUIRE(!zsave, "resblock_fwd: the fused per-block kernel keeps z on chip (pass no zsave)");
      return resblock_fwd_skip(xin, haux, w1, b1, w2, b2, xout, skip, B, T, S, dilation, skip_init, (cudaStream_t)stream);
    }
    WNB_REQUIRE(composed_tc_supported(R, S, Ap, ks), "resblock_fwd: shape R=%d S=%d Ap=%d ks=%d not supported by the "
                "tensor-core paths (use WNB_MATH_FP32)", R, S, Ap, ks);
    if (zsave) return resblock_fwd_composed(p, (cudaStream_t)stream);
    // no z scratch from the caller: a stream-ordered (B,T,R) buffer for the duration of the call
    cudaStream_t st = (cudaStream_t)stream;
    float* z = nullptr;
    WNB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&z), (size_t)B * T * R * sizeof(float), st));
    p.zsave = z;
    const int rc = resblock_fwd_composed(p, st);
    WNB_CUDA(cudaFreeAsync(z, st));
    return rc;
  }
  WNB_REQUIRE(math_mode == WNB_MATH_FP32, "resblock_fwd: unknown math_mode %d", math_mode);
  const size_t smem = sizeof(TileSmem<8>) + (size_t)R * kBsLd * sizeof(float);
  WNB_REQUIRE(smem <= 227 * 1024, "resblock_fwd: n_resch=%d too large for the SIMT path", R);
  if (smem > 48 * 1024) WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(resblock_fwd_simt_kernel), smem));
  dim3 grid(cdiv(T, kBN), B);
  resblock_fwd_simt_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(p);
  WNB_CHECK_LAUNCH("resblock_fwd_simt");
  return WNB_OK;
}

// standalone CausalConv1d forward (wavenet.py:95-121) on channels-last tensors, fp32 FFMA:
//   out[b][t][o] = bias[o] + sum_j sum_c w[o][j*Cin + c] * x[b][t - (ks-1-j)*dilation][c]   (zero for t < 0)
WNB_API int wnb_causal_conv1d_fwd(const float* x, const float* w, const float* bias, float* out, int B, int T, int Cin,
                                  int Cout, int ks, int dilation, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && Cin > 0 && Cout > 0 && ks >= 1 && ks <= 4 && dilation >= 1, "causal_conv1d_fwd: bad shape");
  WNB_REQUIRE(x && w && out, "causal_conv1d_fwd: null pointer");
  NtParams p{};
  p.nseg = ks;
  for (int j = 0; j < ks; j++) p.seg[j] = NtSeg{w + (size_t)j * Cin, ks * Cin, x, Cin, -(ks - 1 - j) * dilation, Cin};
  p.M = Cout; p.T = T; p.B = B; p.bias = bias; p.c = out; p.ldc = Cout;
  return launch_nt(p, (cudaStream_t)stream);
}

WNB_API int wnb_resblock_fwd_supported(int R, int S, int Ap, int ks, int math_mode) {
  if (R <= 0 || S <= 0 || Ap <= 0 || ks < 1) return 0;
  if (math_mode == WNB_MATH_TF32)   // 1 = fused per-block kernel, 2 = composed tensor-core path (zsave scratch)
    return resblock_fwd_skip_supported(R, S, Ap, ks) ? 1 : (composed_tc_supported(R, S, Ap, ks) ? 2 : 0);
  if (math_mode == WNB_MATH_BF16) return composed_tc_supported(R, S, Ap, ks) ? 2 : 0;
  if (math_mode != WNB_MATH_FP32) return 0;
  return (sizeof(TileSmem<8>) + (size_t)R * kBsLd * sizeof(float)) <= 227 * 1024 ? 1 : 0;
}

WNB_API size_t wnb_resblock_bwd_workspace(int B, int T, int R, int S, int Ap, int ks) {
  (void)S; (void)Ap; (void)ks;
  return (size_t)B * T * 3 * R * sizeof(float);  // z (B,T,R) + dpre (B,T,2R)
}

WNB_API int wnb_resblock_bwd(const float* xin, const float* haux, const float* dout, const float* dskip, const float* w1,
                     const float* b1, const float* w1t, const float* w2t, float* dxin, float* dhaux, float* dw1,
                     float* db1, float* dw2, float* db2, void* workspace, int B, int T, int R, int S, int Ap, int ks,
                     int dilation, int math_mode, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && R > 0 && S > 0 && Ap > 0 && ks >= 1 && dilation >= 1, "resblock_bwd: bad shape");
  WNB_REQUIRE(xin && haux && dskip && w1 && b1 && w1t && w2t && dxin && dw1 && db1 && dw2 && db2 && workspace,
              "resblock_bwd: null pointer");
  WNB_REQUIRE(math_mode == WNB_MATH_FP32 || math_mode == WNB_MATH_TF32 || math_mode == WNB_MATH_BF16,
              "resblock_bwd: unknown math_mode %d", math_mode);
  WNB_REQUIRE(math_mode != WNB_MATH_BF16 || composed_tc_supported(R, S, Ap, ks), "resblock_bwd: shape R=%d S=%d Ap=%d "
              "ks=%d not supported by the bf16 tensor-core path (use WNB_MATH_TF32 or WNB_MATH_FP32)", R, S, Ap, ks);
  cudaStream_t st = (cudaStream_t)stream;
  float* z = (float*)workspace;
  float* dpre = z + (size_t)B * T * R;
  const int K1 = ks * R + Ap, M2 = R + S;
  int rc;
  const bool tc_fused_shape = math_mode == WNB_MATH_TF32 && R == 64 && ks == 2 && Ap == 32 && S % 32 == 0;
  const bool bf16 = math_mode == WNB_MATH_BF16;
  if (bf16 || (math_mode == WNB_MATH_TF32 && !tc_fused_shape && composed_tc_supported(R, S, Ap, ks))) {
    // ---------------- composed tensor-core backward for general shapes (tf32, or bf16 operands) ----------------
    Bf16Weights bwt;
    const Bf16Weights* bw = nullptr;
    if (bf16) {
      if ((rc = to_bf16_weights(bwt, {{w1, (int64_t)2 * R * K1}, {w1t, (int64_t)K1 * 2 * R}, {w2t, (int64_t)R * M2}}, st)) !=
          WNB_OK)
        return rc;
      bw = &bwt;
    }
    float* dz = dxin;   // (B,T,R) scratch until the dX GEMM overwrites it
    const NtTcOpts opl = plain_opts(R);
    if (dout) {
      NtTcSeg sz[2] = {{dout, R, 0, R, w2t, R, R + S, 0, 0}, {dskip, S, 0, S, w2t, R, R + S, R, 0}};
      Bf16Weights::apply(bw, sz, 2);
      if ((rc = gemm_nt_tc(sz, 2, R / opl.n_blocks, dz, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr,
                           nullptr, 0, 0, nullptr, &opl)) != WNB_OK)
        return rc;
    } else {
      NtTcSeg sz[1] = {{dskip, S, 0, S, w2t, R, R + S, R, 0}};
      Bf16Weights::apply(bw, sz, 1);
      if ((rc = gemm_nt_tc(sz, 1, R / opl.n_blocks, dz, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr,
                           nullptr, 0, 0, nullptr, &opl)) != WNB_OK)
        return rc;
    }
    NtTcSeg sg[4];
    int ns = 0;
    for (int j = 0; j < ks; j++) sg[ns++] = NtTcSeg{xin, R, -(ks - 1 - j) * dilation, R, w1, 2 * R, K1, j * R, 0};
    sg[ns++] = NtTcSeg{haux, Ap, 0, Ap, w1, 2 * R, K1, ks * R, 0};
    Bf16Weights::apply(bw, sg, ns);
    const int GC = composed_gc(R);
        for (int c0 = 0; c0 < R; c0 += GC) {   // gate recompute + z + dpre, GC gate channels per launch
      const NtTcGate g{2, c0, R, b1 + c0, b1 + R + c0, dz, dpre};
      if ((rc = gemm_nt_tc(sg, ns, 2 * GC, z, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr, nullptr, 0,
                           0, &g)) != WNB_OK)
        return rc;
    }
    {  // dxin = dout + sum_j dpre(t + (ks-1-j)d) W1[:, tap j]
      NtTcSeg sx[3];
      for (int j = 0; j < ks; j++) sx[j] = NtTcSeg{dpre, 2 * R, (ks - 1 - j) * dilation, 2 * R, w1t, K1, 2 * R, 0, j * R};
      Bf16Weights::apply(bw, sx, ks);
      if ((rc = gemm_nt_tc(sx, ks, R / opl.n_blocks, dxin, R, nullptr, nullptr, 0, dout, R, 0, 0, B, T, st, nullptr, nullptr,
                           nullptr, 0, 0, nullptr, &opl)) != WNB_OK)
        return rc;
    }
    if (dhaux) {
      NtTcSeg sh[1] = {{dpre, 2 * R, 0, 2 * R, w1t, K1, 2 * R, 0, ks * R}};
      Bf16Weights::apply(bw, sh, 1);
      if ((rc = gemm_nt_tc(sh, 1, Ap, dhaux, Ap, nullptr, nullptr, 0, nullptr, 0, 0, 1, B, T, st)) != WNB_OK) return rc;
    }
    // dW1 = dpre^T [x taps | aux]  (+ db1), dW2 = [dout | dskip]^T z  (+ db2)
    for (int j = 0; j < ks; j++)
      if ((rc = wgrad_tc_concat(dpre, 2 * R, nullptr, 0, 2 * R, xin, R, R, -(ks - 1 - j) * dilation, dw1 + j * R, K1,
                                j == 0 ? db1 : nullptr, B, T, st, bf16)) != WNB_OK)
        return rc;
    if ((rc = wgrad_tc_concat(dpre, 2 * R, nullptr, 0, 2 * R, haux, Ap, Ap, 0, dw1 + ks * R, K1, nullptr, B, T, st, bf16)) !=
        WNB_OK)
      return rc;
    if (dout) return wgrad_tc_concat(dout, R, dskip, S, R + S, z, R, R, 0, dw2, R, db2, B, T, st, bf16);
    return wgrad_tc_concat(dskip, S, nullptr, 0, S, z, R, R, 0, dw2 + (size_t)R * R, R, db2 + R, B, T, st, bf16);
  }
  const bool tc_bwd = tc_fused_shape;
  if (tc_bwd) {
    // dz[t][c] = sum_r w2[r][c] dout[t][r] + sum_s w2[R+s][c] dskip[t][s]   (w2t: rows c, cols o)
    float* dz = dxin;   // dxin is not produced until the dX GEMM below: use it as the (B,T,64) scratch for dz
    if (dout) {
      const NtTcSeg sz[2] = {{dout, R, 0, R, w2t, R, R + S, 0, 0}, {dskip, S, 0, S, w2t, R, R + S, R, 0}};
      if ((rc = gemm_nt_tc(sz, 2, R, dz, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st)) != WNB_OK) return rc;
    } else {
      const NtTcSeg sz[1] = {{dskip, S, 0, S, w2t, R, R + S, R, 0}};
      if ((rc = gemm_nt_tc(sz, 1, R, dz, R, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st)) != WNB_OK) return rc;
    }
    // gate recompute (pre = W1 [x(t-d) | x(t) | aux]) fused with z and dpre in the epilogue
    const NtTcSeg sg[3] = {{xin, R, -dilation, R, w1, 2 * R, K1, 0, 0}, {xin, R, 0, R, w1, 2 * R, K1, R, 0},
                           {haux, Ap, 0, Ap, w1, 2 * R, K1, 2 * R, 0}};
    if ((rc = gemm_nt_tc(sg, 3, 2 * R, z, R, b1, nullptr, 0, nullptr, 0, 0, 0, B, T, st, dz, dpre)) != WNB_OK) return rc;
  } else {
    BwdGateParams g{xin, haux, dout, dskip, w1, b1, w2t, z, dpre, B, T, R, S, Ap, ks, dilation};
    dim3 grid(cdiv(T, kBN), B, cdiv(R, 64));
    resblock_bwd_gate_kernel<<<grid, kThreads, 0, st>>>(g);
    WNB_CHECK_LAUNCH("resblock_bwd_gate");
  }
  if (tc_bwd) {
    // dxin = dout + dpre(t+d) W1[:, tap0] + dpre(t) W1[:, tap1]   and   dhaux += dpre(t) W1[:, aux]
    // (w1t rows: 0-63 tap0, 64-127 tap1, 128-159 aux).  One GEMM with N = 96: the tap-0 segment sees w1t as a
    // 64-row matrix, so its rows 64-95 are TMA zero fill and only tap 1 feeds the aux columns.
    if (dhaux) {
      const NtTcSeg sx[2] = {{dpre, 2 * R, dilation, 2 * R, w1t, R, 2 * R, 0, 0},
                             {dpre, 2 * R, 0, 2 * R, w1t, K1, 2 * R, 0, R}};
      if ((rc = gemm_nt_tc(sx, 2, R + Ap, dxin, R, nullptr, nullptr, 0, dout, R, 0, 0, B, T, st, nullptr, nullptr,
                           dhaux, Ap, R)) != WNB_OK)
        return rc;
    } else {
      const NtTcSeg sx[2] = {{dpre, 2 * R, dilation, 2 * R, w1t, K1, 2 * R, 0, 0},
                             {dpre, 2 * R, 0, 2 * R, w1t, K1, 2 * R, 0, R}};
      if ((rc = gemm_nt_tc(sx, 2, R, dxin, R, nullptr, nullptr, 0, dout, R, 0, 0, B, T, st)) != WNB_OK) return rc;
    }
  } else {
  {  // dxin[t][c] = dout[t][c] + sum_j sum_o w1[o][j*R+c] * dpre[t+(ks-1-j)d][o]
    NtParams p{};
    p.nseg = ks;
    WNB_REQUIRE(ks <= 4, "resblock_bwd: kernel_size > 4 unsupported");
    for (int j = 0; j < ks; j++)
      p.seg[j] = NtSeg{w1t + (size_t)j * R * 2 * R, 2 * R, dpre, 2 * R, (ks - 1 - j) * dilation, 2 * R};
    p.M = R; p.T = T; p.B = B; p.bias = nullptr; p.c = dxin; p.ldc = R;
    p.add = dout; p.ldadd = R; p.mask = nullptr; p.ldmask = 0; p.relu_b = 0; p.relu_out = 0; p.accumulate = 0;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  if (dhaux) {  // dhaux[t][a] += sum_o w1[o][ks*R+a] * dpre[t][o]
    NtParams p{};
    p.nseg = 1;
    p.seg[0] = NtSeg{w1t + (size_t)ks * R * 2 * R, 2 * R, dpre, 2 * R, 0, 2 * R};
    p.M = Ap; p.T = T; p.B = B; p.bias = nullptr; p.c = dhaux; p.ldc = Ap;
    p.add = nullptr; p.mask = nullptr; p.relu_b = 0; p.relu_out = 0; p.accumulate = 1;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  }
  // weight gradients
  const bool tc_wgrad = math_mode == WNB_MATH_TF32 && R == 64 && ks == 2 && Ap == 32 && S % 32 == 0;
  if (tc_wgrad) {
    {  // dW1 (128 x 160) += dpre^T [x(t-d) | x(t) | aux(t)],  db1 = column sums of dpre
      const WgOperand a[1] = {{dpre, 2 * R, 0, 4, 0}};
      const WgOperand b[3] = {{xin, R, 0, 2, -dilation}, {xin, R, 0, 2, 0}, {haux, Ap, 0, 1, 0}};
      if ((rc = wgrad_tc(a, 1, b, 3, dw1, K1, 128, db1, B, T, st)) != WNB_OK) return rc;
    }
    // dW2 (R+S x R) += [dout | dskip]^T z,  db2 = column sums of [dout | dskip]: row blocks of 128, up to 5 per
    // launch (z and dskip are streamed once, through L2)
    const WgOperand bz[1] = {{z, R, 0, 2, 0}};
    const int row_first = dout ? 0 : R;
    WgBlock blk[5];
    int nblk = 0;
    for (int r0 = row_first; r0 < R + S; r0 += 128) {
      WgBlock& bk = blk[nblk];
      bk.m_valid = (R + S - r0) < 128 ? (R + S - r0) : 128;
      bk.c = dw2 + (size_t)r0 * R;
      bk.db = db2 + r0;
      if (r0 == 0) {
        bk.nops = 2;
        bk.ops[0] = WgOperand{dout, R, 0, 2, 0};
        bk.ops[1] = WgOperand{dskip, S, 0, 2, 0};
      } else {
        bk.nops = 1;
        bk.ops[0] = WgOperand{dskip, S, r0 - R, 4, 0};
      }
      if (++nblk == 5 || r0 + 128 >= R + S) {
        if ((rc = wgrad_tc_blocks(blk, nblk, bz, 1, R, B, T, st)) != WNB_OK) return rc;
        nblk = 0;
      }
    }
    return WNB_OK;
  }
  for (int j = 0; j < ks; j++) {
    TnParams p{dpre, 2 * R, 2 * R, xin, R, R, -(ks - 1 - j) * dilation, 0, dw1, K1, j * R, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(2 * R, 128) * cdiv(R, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
  }
  {
    TnParams p{dpre, 2 * R, 2 * R, haux, Ap, Ap, 0, 0, dw1, K1, ks * R, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(2 * R, 128) * cdiv(Ap, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
  }
  if ((rc = launch_colsum(dpre, 2 * R, 2 * R, (int64_t)B * T, db1, st)) != WNB_OK) return rc;
  if (dout) {
    TnParams p{dout, R, R, z, R, R, 0, 0, dw2, R, 0, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(R, 128) * cdiv(R, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
    if ((rc = launch_colsum(dout, R, R, (int64_t)B * T, db2, st)) != WNB_OK) return rc;
  }
  {
    TnParams p{dskip, S, S, z, R, R, 0, 0, dw2 + (size_t)R * R, R, 0, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(S, 128) * cdiv(R, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
    if ((rc = launch_colsum(dskip, S, S, (int64_t)B * T, db2 + R, st)) != WNB_OK) return rc;
  }
  (void)M2;
  return WNB_OK;
}

WNB_API int wnb_post_fwd(float* skip, const float* wp1, const float* bp1, const float* wp2, const float* bp2,
                 float* r1, float* logits, int B, int T, int S, int Q, int math_mode, int skip_rectified,
                 void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && S > 0 && Q > 0, "post_fwd: bad shape");
  WNB_REQUIRE(skip && wp1 && bp1 && wp2 && bp2 && r1 && logits, "post_fwd: null pointer (r1 scratch is required)");
  WNB_REQUIRE(math_mode == WNB_MATH_FP32 || math_mode == WNB_MATH_TF32 || math_mode == WNB_MATH_BF16,
              "post_fwd: unknown math_mode %d", math_mode);
  WNB_REQUIRE(math_mode != WNB_MATH_BF16 || (nt_tc_n_ok(S) && nt_tc_n_ok(Q)),
              "post_fwd: S=%d Q=%d not supported by the bf16 tensor-core path", S, Q);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((math_mode == WNB_MATH_TF32 || math_mode == WNB_MATH_BF16) && nt_tc_n_ok(S) && nt_tc_n_ok(Q)) {
    // rectify the skip sum in place (its sign pattern, all the backward needs, is unchanged), then two
    // tensor-core GEMMs with fused bias / ReLU epilogues
    Bf16Weights bwt;
    const Bf16Weights* bw = nullptr;
    if (math_mode == WNB_MATH_BF16) {
      if ((rc = to_bf16_weights(bwt, {{wp1, (int64_t)S * S}, {wp2, (int64_t)Q * S}}, st)) != WNB_OK) return rc;
      bw = &bwt;
    }
    const int64_t n4 = (int64_t)B * T * S / 4;
    if (!skip_rectified) {
      relu_inplace_kernel<<<device_sms() * 8, 256, 0, st>>>(reinterpret_cast<float4*>(skip), n4);
      WNB_CHECK_LAUNCH("relu_inplace");
    }
    NtTcSeg s1[1] = {{skip, S, 0, S, wp1, S, S, 0, 0}};
    Bf16Weights::apply(bw, s1, 1);
    if (post_split(S)) {   // two 256-column blocks: double-buffered accumulators, epilogue overlapped with the next tile
      const NtTcOpts o{2};
      if ((rc = gemm_nt_tc(s1, 1, S / 2, r1, S, bp1, nullptr, 0, nullptr, 0, 1, 0, B, T, st, nullptr, nullptr, nullptr, 0, 0,
                           nullptr, &o)) != WNB_OK)
        return rc;
    } else if ((rc = gemm_nt_tc(s1, 1, S, r1, S, bp1, nullptr, 0, nullptr, 0, 1, 0, B, T, st)) != WNB_OK) return rc;
    NtTcSeg s2[1] = {{r1, S, 0, S, wp2, Q, S, 0, 0}};
    Bf16Weights::apply(bw, s2, 1);
    const NtTcOpts o2{1};
    return gemm_nt_tc(s2, 1, Q, logits, Q, bp2, nullptr, 0, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr, nullptr, 0, 0,
                      nullptr, &o2);
  }
  // (skip_rectified: the FFMA GEMM below applies ReLU to its B operand anyway, and ReLU is idempotent)
  {  // r1 = relu(wp1 * relu(skip) + bp1)
    NtParams p{};
    p.nseg = 1; p.seg[0] = NtSeg{wp1, S, skip, S, 0, S};
    p.M = S; p.T = T; p.B = B; p.bias = bp1; p.c = r1; p.ldc = S; p.relu_b = 1; p.relu_out = 1;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  {  // logits = wp2 * r1 + bp2
    NtParams p{};
    p.nseg = 1; p.seg[0] = NtSeg{wp2, S, r1, S, 0, S};
    p.M = Q; p.T = T; p.B = B; p.bias = bp2; p.c = logits; p.ldc = Q;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  return WNB_OK;
}

WNB_API int wnb_post_bwd(const float* skip, const float* r1, const float* dlogits, const float* wp1t, const float* wp2t,
                 float* dskip, float* dwp1, float* dbp1, float* dwp2, float* dbp2, float* workspace, int B, int T,
                 int S, int Q, int math_mode, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && S > 0 && Q > 0, "post_bwd: bad shape");
  WNB_REQUIRE(skip && r1 && dlogits && wp1t && wp2t && dskip && dwp1 && dbp1 && dwp2 && dbp2 && workspace,
              "post_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  WNB_REQUIRE(math_mode == WNB_MATH_FP32 || math_mode == WNB_MATH_TF32 || math_mode == WNB_MATH_BF16,
              "post_bwd: unknown math_mode %d", math_mode);
  WNB_REQUIRE(math_mode != WNB_MATH_BF16 || (nt_tc_n_ok(S) && nt_tc_n_ok(Q)),
              "post_bwd: S=%d Q=%d not supported by the bf16 tensor-core path", S, Q);
  float* dh1 = workspace;  // (B,T,S)
  int rc;
  const bool bf16 = math_mode == WNB_MATH_BF16;
  if ((math_mode == WNB_MATH_TF32 || bf16) && nt_tc_n_ok(S) && nt_tc_n_ok(Q)) {
    // (skip was rectified in place by the tensor-core forward, so it doubles as relu(skip) and as the sign mask)
    Bf16Weights bwt;
    const Bf16Weights* bw = nullptr;
    if (bf16) {
      if ((rc = to_bf16_weights(bwt, {{wp2t, (int64_t)S * Q}, {wp1t, (int64_t)S * S}}, st)) != WNB_OK) return rc;
      bw = &bwt;
    }
    NtTcSeg s1[1] = {{dlogits, Q, 0, Q, wp2t, S, Q, 0, 0}};
    NtTcSeg s2[1] = {{dh1, S, 0, S, wp1t, S, S, 0, 0}};
    Bf16Weights::apply(bw, s1, 1);
    Bf16Weights::apply(bw, s2, 1);
    if (post_split(S)) {
      const NtTcOpts o{2};
      if ((rc = gemm_nt_tc(s1, 1, S / 2, dh1, S, nullptr, r1, S, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr, nullptr, 0, 0,
                           nullptr, &o)) != WNB_OK)
        return rc;
      if ((rc = gemm_nt_tc(s2, 1, S / 2, dskip, S, nullptr, skip, S, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr, nullptr, 0,
                           0, nullptr, &o)) != WNB_OK)
        return rc;
    } else {
      if ((rc = gemm_nt_tc(s1, 1, S, dh1, S, nullptr, r1, S, nullptr, 0, 0, 0, B, T, st)) != WNB_OK) return rc;
      if ((rc = gemm_nt_tc(s2, 1, S, dskip, S, nullptr, skip, S, nullptr, 0, 0, 0, B, T, st)) != WNB_OK) return rc;
    }
    // 2 launches of (2 M-blocks x 128-column groups) for dWp1: a squarer tile than 4 M-blocks x 64 columns; same-box
    // A/B (two repetitions each): 8.90 / 8.95 ms per step against 8.97 / 8.97 (WNB_POST_WG_OLD=1 selects the old split)
    static const bool old_split = [] { const char* e = getenv("WNB_POST_WG_OLD"); return e && e[0] == '1'; }();
    if (bf16) {
      if ((rc = wgrad_tc_concat(dlogits, Q, nullptr, 0, Q, r1, S, S, 0, dwp2, S, dbp2, B, T, st, true)) != WNB_OK) return rc;
      return wgrad_tc_concat(dh1, S, nullptr, 0, S, skip, S, S, 0, dwp1, S, dbp1, B, T, st, true);
    }
    if (old_split) {
      if ((rc = wgrad_tc_split(dlogits, Q, Q, r1, S, S, dwp2, S, dbp2, B, T, st)) != WNB_OK) return rc;
      return wgrad_tc_split(dh1, S, S, skip, S, S, dwp1, S, dbp1, B, T, st);
    }
    if ((rc = wgrad_tc_concat(dlogits, Q, nullptr, 0, Q, r1, S, S, 0, dwp2, S, dbp2, B, T, st)) != WNB_OK) return rc;
    return wgrad_tc_concat(dh1, S, nullptr, 0, S, skip, S, S, 0, dwp1, S, dbp1, B, T, st);
  }
  {  // dh1[t][c] = (sum_q wp2[q][c] dlogits[t][q]) * (r1 > 0)
    NtParams p{};
    p.nseg = 1; p.seg[0] = NtSeg{wp2t, Q, dlogits, Q, 0, Q};
    p.M = S; p.T = T; p.B = B; p.c = dh1; p.ldc = S; p.mask = r1; p.ldmask = S;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  {  // dskip[t][c] = (sum_o wp1[o][c] dh1[t][o]) * (skip > 0)
    NtParams p{};
    p.nseg = 1; p.seg[0] = NtSeg{wp1t, S, dh1, S, 0, S};
    p.M = S; p.T = T; p.B = B; p.c = dskip; p.ldc = S; p.mask = skip; p.ldmask = S;
    if ((rc = launch_nt(p, st)) != WNB_OK) return rc;
  }
  {  // dwp2[q][c] += sum_t dlogits[t][q] * r1[t][c]
    TnParams p{dlogits, Q, Q, r1, S, S, 0, 0, dwp2, S, 0, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(Q, 128) * cdiv(S, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
    if ((rc = launch_colsum(dlogits, Q, Q, (int64_t)B * T, dbp2, st)) != WNB_OK) return rc;
  }
  {  // dwp1[o][c] += sum_t dh1[t][o] * relu(skip[t][c])
    TnParams p{dh1, S, S, skip, S, S, 0, 1, dwp1, S, 0, T, B, 0};
    p.tchunk = pick_tchunk(B, T, cdiv(S, 128) * cdiv(S, kBN));
    if ((rc = launch_tn(p, st)) != WNB_OK) return rc;
    if ((rc = launch_colsum(dh1, S, S, (int64_t)B * T, dbp1, st)) != WNB_OK) return rc;
  }
  return WNB_OK;
}

}  // extern "C"
