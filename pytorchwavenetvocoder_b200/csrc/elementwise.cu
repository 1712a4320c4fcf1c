// elementwise.cu -- mu-law codec, front embedding gather, aux up-sampling and the fused
// cross-entropy (+gradient) kernel.  All HBM-bound streaming kernels: coalesced channels-last rows,
// float4 where the row width allows, grids sized in multiples of the SM count by grid-stride loops.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "common.cuh"

namespace wnb {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n); }
bool pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("WNB_PDL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on == 1;
}

// ---- per-device / per-stream launch state ----
static std::mutex g_state_mu;
int device_sms() {
  static int sms[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  std::lock_guard<std::mutex> lk(g_state_mu);
  if (!sms[dev] && cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms[dev] = 132;
  return sms[dev];
}
cudaError_t ensure_dynamic_smem(const void* func, size_t bytes) {
  static std::map<std::pair<int, const void*>, size_t> done;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(g_state_mu);
  size_t& have = done[std::make_pair(dev, func)];
  if (bytes > have) {
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    have = bytes;
  }
  return cudaSuccess;
}
unsigned int* sched_counters(cudaStream_t st) {
  static std::map<std::pair<int, cudaStream_t>, unsigned int*> slots;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(g_state_mu);
  unsigned int*& p = slots[std::make_pair(dev, st)];
  if (!p) {
    if (cudaMalloc(&p, 256) != cudaSuccess) { p = nullptr; return nullptr; }
    if (cudaMemset(p, 0, 256) != cudaSuccess) { cudaFree(p); p = nullptr; return nullptr; }
  }
  return p;
}

void* scratch_buffer(cudaStream_t st, int slot, size_t bytes) {
  // A buffer that has been outgrown is kept, not freed: work already queued on the stream, or another host thread that
  // obtained it, may still use it.  Sizes grow geometrically, so what is kept is less than the live buffer.
  struct Buf { void* p; size_t n; };
  static std::mutex mu;
  static std::map<std::tuple<int, cudaStream_t, int>, Buf> bufs;
  static std::vector<void*> retired;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  Buf& b = bufs[std::make_tuple(dev, st, slot)];
  if (b.n < bytes) {
    const size_t n = bytes > 2 * b.n ? bytes : 2 * b.n;
    void* p = nullptr;
    if (cudaMalloc(&p, n) != cudaSuccess) return nullptr;
    if (b.p) retired.push_back(b.p);
    b.p = p; b.n = n;
  }
  return b.p;
}

// ---- per-launch event timing (off by default; bench.py switches it on for the timed region) ----
struct ProfRec { int kind; cudaEvent_t e0, e1; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof_recs;      // records of the current session
static std::vector<cudaEvent_t> g_prof_pool;  // recycled events
static cudaEvent_t prof_event() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
void prof_begin(int kind, cudaStream_t st) {
  if (!g_prof_on) return;
  ProfRec r{kind, prof_event(), prof_event()};
  cudaEventRecord(r.e0, st);
  g_prof_recs.push_back(r);
}
void prof_end(int kind, cudaStream_t st) {
  if (!g_prof_on || g_prof_recs.empty() || g_prof_recs.back().kind != kind) return;
  cudaEventRecord(g_prof_recs.back().e1, st);
}

static int grid_for(int64_t work_items, int threads) {
  int64_t blocks = (work_items + threads - 1) / threads;
  const int64_t cap = (int64_t)device_sms() * 16;  // 16 resident 256-thread CTAs per SM is plenty for streaming kernels
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// ------------------------------------------------------------------------------------------------
// mu-law (wavenet.py:17-30, 33-47).  Bit exactness with numpy: numpy evaluates
//   fx = sign(x) * log(1 + mu*|x|) / log(1 + mu);  floor((fx + 1) / 2 * mu + 0.5)
// elementwise; for float32 input sign/abs/log stay float32 and the division by the numpy float64
// scalar np.log(1 + mu) promotes the rest to float64 (NEP 50).  We evaluate the same expression tree
// in the same dtypes with FMA contraction disabled.  The float32 log is computed correctly rounded
// (double log, round to float).  numpy's own SIMD float32 log is NOT correctly rounded (~4 % of
// inputs differ by 1 ulp, CPU-dispatch dependent), which only matters for float32 inputs sitting
// within 1 ulp of a quantiser edge: there the reference's answer is build dependent and ours can
// differ by one code.  On the whole PCM-16 domain (s/32768, what sf.read(dtype=float32) yields for
// the recipes' wavs, bin/train.py:121) and on dense grids the result is bit exact
// (tests/golden/mulaw.npz, tests/test_gpu_parity.py).
// ------------------------------------------------------------------------------------------------
__global__ void mulaw_encode_f32_kernel(const float* __restrict__ x, int64_t* __restrict__ y, int64_t n,
                                        float mu, double log1pmu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float sgn = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
    // float32 part: sign(x) * log(1 + mu*|x|)   (numpy keeps float32 here)
    const float arg = __fadd_rn(1.0f, __fmul_rn(mu, fabsf(v)));
    const float lg = (float)log((double)arg);  // correctly rounded float32 log
    const float num = __fmul_rn(sgn, lg);
    // "/ np.log(1 + mu)" divides by a numpy float64 scalar: NEP-50 promotes the rest to float64
    const double fx = __ddiv_rn((double)num, log1pmu);
    const double q = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(fx, 1.0), 2.0), (double)mu), 0.5);
    y[i] = (int64_t)floor(q);
  }
}

__global__ void mulaw_encode_f64_kernel(const double* __restrict__ x, int64_t* __restrict__ y, int64_t n,
                                        double mu, double log1pmu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = x[i];
    const double sgn = (v > 0.) ? 1. : ((v < 0.) ? -1. : 0.);
    const double arg = __dadd_rn(1.0, __dmul_rn(mu, fabs(v)));
    const double fx = __ddiv_rn(__dmul_rn(sgn, log(arg)), log1pmu);
    const double q = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(fx, 1.0), 2.0), mu), 0.5);
    y[i] = (int64_t)floor(q);
  }
}

// decode: the input domain is the mu integer codes, so the launcher evaluates the reference
// expression  fx = (y - 0.5) / mu * 2 - 1 ; x = sign(fx) / mu * ((1 + mu) ** |fx| - 1)  once per code on
// the host with the correctly rounded libm pow and the kernel is a table gather.  (numpy's float64
// power is SVML on AVX-512 hosts and libm elsewhere; the two differ by 1 ulp in 11 of 256 codes, so the
// reference itself is only defined up to 1 ulp here; after the PCM_16 quantisation of
// bin/decode.py:319 all variants are identical.)
struct MulawTable { double v[256]; };

__global__ void mulaw_decode_f64_kernel(const int64_t* __restrict__ y, double* __restrict__ x, int64_t n,
                                        double mu, int nmu, const MulawTable tab) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t yi = y[i];
    if (yi >= 0 && yi < nmu && nmu <= 256) {
      x[i] = tab.v[yi];
    } else {
      const double fx = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn((double)yi, -0.5), mu), 2.0), -1.0);
      const double sgn = (fx > 0.) ? 1. : ((fx < 0.) ? -1. : 0.);
      const double pw = pow(1.0 + mu, fabs(fx));
      x[i] = __dmul_rn(__ddiv_rn(sgn, mu), __dadd_rn(pw, -1.0));
    }
  }
}

// codes -> PCM_16 for a whole batch (decode driver, bin/decode.py:318-319: decode_mu_law + write "PCM_16"): the input
// domain is the mu integer codes, so the host evaluates decode + quantisation once per code and this is a 2-byte gather
__global__ void lut_i16_kernel(const int32_t* __restrict__ idx, const int16_t* __restrict__ table, int16_t* __restrict__ out,
                               int64_t n, int ntab) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int v = idx[i] % ntab;
    if (v < 0) v += ntab;
    out[i] = __ldg(table + v);
  }
}

// ------------------------------------------------------------------------------------------------
// front embedding gather (wavenet.py:78-92 OneHot + :513-516 causal conv)
//   out[b][t][r] = bias[r] + sum_k wf[k][x[b][t-(ks-1-k)] mod Q][r]   (missing history: zero)
// One thread per 4 channels of one (b,t) row; rows are 4R bytes contiguous -> coalesced stores.
// ------------------------------------------------------------------------------------------------
__global__ void front_embed_fwd_kernel(const int64_t* __restrict__ x, const float* __restrict__ wf,
                                       const float* __restrict__ bias, float* __restrict__ out, int B, int T,
                                       int Q, int R, int ks) {
  const int64_t total = (int64_t)B * T * R;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % R);
    const int64_t bt = i / R;
    const int t = (int)(bt % T);
    float v = bias[r];
    for (int k = 0; k < ks; k++) {
      const int tt = t - (ks - 1 - k);
      if (tt >= 0) {
        int64_t q = x[bt - (ks - 1 - k)] % Q;
        if (q < 0) q += Q;
        v += __ldg(wf + ((size_t)k * Q + q) * R + r);
      }
    }
    out[i] = v;
  }
}
// R % 4 == 0: one thread per 4 channels (16-byte gathers from the L2-resident table, 16-byte coalesced stores), 32-bit
// index arithmetic on the row, no per-element 64-bit division
__global__ void __launch_bounds__(256) front_embed_fwd_v4_kernel(const int64_t* __restrict__ x, const float4* __restrict__ wf,
                                                                 const float4* __restrict__ bias, float4* __restrict__ out,
                                                                 int B, int T, int Q, int R4, int ks) {
  const int rows_per_blk = blockDim.x / R4;                 // host guarantees blockDim.x % R4 == 0
  const int lr = threadIdx.x / R4, r4 = threadIdx.x - lr * R4;
  const int64_t nrows = (int64_t)B * T;
  const float4 bv = __ldg(bias + r4);
  for (int64_t row = (int64_t)blockIdx.x * rows_per_blk + lr; row < nrows; row += (int64_t)gridDim.x * rows_per_blk) {
    const int t = (int)(row % T);
    float4 v = bv;
    for (int k = 0; k < ks; k++) {
      const int s_ = ks - 1 - k;
      if (t - s_ >= 0) {
        int64_t q = x[row - s_] % Q;
        if (q < 0) q += Q;
        const float4 w = __ldg(wf + ((size_t)k * Q + q) * R4 + r4);
        v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
      }
    }
    out[row * R4 + r4] = v;
  }
}

// dwf[k][q][r] += sum of dout[b][t][r] over the rows whose tap-k token x[b][t-(ks-1-k)] is q.  A scatter by token:
// instead of atomics (whose order depends on scheduling), block q scans all rows and owns row q of every tap's table,
// so each sum is taken in one fixed order.  Threads: `lanes` time lanes x Rv channel groups of V floats; lane l takes the
// rows l, l + lanes, ... and the lanes are added in lane order.  The tap with no shift sees every row exactly once, so
// its per-token sums (qpart) add up to the bias gradient.
// tok[row] = x[row] mod Q in [0, Q): computed once per call instead of in every block of the scan below
__global__ void token_kernel(const int64_t* __restrict__ x, int* __restrict__ tok, int64_t n, int Q) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t q = x[i] % Q;
    tok[i] = (int)(q < 0 ? q + Q : q);
  }
}
template <int V>
__global__ void __launch_bounds__(512) front_embed_bwd_kernel(const int* __restrict__ tok, const float* __restrict__ dout,
                                                              float* __restrict__ dwf, float* __restrict__ qpart, int B, int T,
                                                              int Q, int Rv, int ks) {
  typedef typename std::conditional<V == 4, float4, float>::type vec;
  constexpr int kMaxKs = 4;
  const int q = blockIdx.x;
  const int lanes = blockDim.x / Rv;
  const int lr = threadIdx.x / Rv, rv = threadIdx.x - lr * Rv;
  const vec* dv = reinterpret_cast<const vec*>(dout);
  float acc[kMaxKs][V];
#pragma unroll
  for (int k = 0; k < kMaxKs; k++)
#pragma unroll
    for (int i = 0; i < V; i++) acc[k][i] = 0.f;
  for (int b = 0; b < B; b++)
  for (int t = lr; t < T; t += lanes) {
    const int64_t row = (int64_t)b * T + t;
#pragma unroll
    for (int k = 0; k < kMaxKs; k++) {
      if (k >= ks) break;
      const int s_ = ks - 1 - k;
      if (t - s_ < 0 || __ldg(tok + row - s_) != q) continue;
      const vec g = __ldg(dv + row * Rv + rv);
      const float* gf = reinterpret_cast<const float*>(&g);
#pragma unroll
      for (int i = 0; i < V; i++) acc[k][i] += gf[i];
    }
  }
  __shared__ float red[512 * V];
  for (int k = 0; k < ks && k < kMaxKs; k++) {
#pragma unroll
    for (int i = 0; i < V; i++) red[threadIdx.x * V + i] = acc[k][i];
    __syncthreads();
    if (lr == 0) {
      float sum[V];
#pragma unroll
      for (int i = 0; i < V; i++) sum[i] = 0.f;
      for (int l = 0; l < lanes; l++)
#pragma unroll
        for (int i = 0; i < V; i++) sum[i] += red[(l * Rv + rv) * V + i];
      float* dst = dwf + ((size_t)k * Q + q) * Rv * V + (size_t)rv * V;
#pragma unroll
      for (int i = 0; i < V; i++) dst[i] += sum[i];
      if (k == ks - 1)
#pragma unroll
        for (int i = 0; i < V; i++) qpart[((size_t)q * Rv + rv) * V + i] = sum[i];
    }
    __syncthreads();
  }
}
// Chunked form of the same sums, for tables that fit in shared memory: block c owns rows [c * chunk, (c + 1) * chunk)
// and builds its own (ks, Q, R) table there.  Thread (qg, rv) owns the entries of the tokens q with q % QG == qg and
// channel group rv, and walks the block's rows in order, so every entry is summed in one fixed order without atomics;
// the per-chunk tables are then added in chunk order (front_embed_reduce_kernel).
__global__ void __launch_bounds__(256) front_embed_bwd_chunk_kernel(const int* __restrict__ tok, const float4* __restrict__ dout,
                                                                    float* __restrict__ part, int B, int T, int Q, int R4, int ks,
                                                                    int64_t chunk) {
  extern __shared__ float4 tab[];                    // [ks][Q][R4]
  const int QG = blockDim.x / R4;
  const int qg = threadIdx.x / R4, rv = threadIdx.x - qg * R4;
  const int n4 = ks * Q * R4;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) tab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  const int64_t nrows = (int64_t)B * T;
  const int64_t row0 = (int64_t)blockIdx.x * chunk;
  const int64_t row1 = row0 + chunk < nrows ? row0 + chunk : nrows;
  int t = (int)(row0 % T);
  for (int64_t row = row0; row < row1; row++) {
    for (int k = 0; k < ks; k++) {
      const int s_ = ks - 1 - k;
      if (t - s_ < 0) continue;
      const int q = __ldg(tok + row - s_);
      if (q % QG != qg) continue;
      const float4 g = __ldg(dout + row * R4 + rv);
      float4& e = tab[((size_t)k * Q + q) * R4 + rv];
      e.x += g.x; e.y += g.y; e.z += g.z; e.w += g.w;
    }
    if (++t == T) t = 0;
  }
  __syncthreads();
  float4* dst = reinterpret_cast<float4*>(part) + (size_t)blockIdx.x * n4;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = tab[i];
}
// dwf[i] += sum over chunks c (in order) of part[c][i]; the last tap's sums also go to qpart (for the bias gradient)
__global__ void front_embed_reduce_kernel(const float* __restrict__ part, float* __restrict__ dwf, float* __restrict__ qpart,
                                          int nchunks, int n, int last0) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < nchunks; c++) s += part[(size_t)c * n + i];
    dwf[i] += s;
    if (i >= last0) qpart[i - last0] = s;
  }
}
// out[r] += sum over rows j = 0 .. n-1 (in that order) of part[j * ld + r], r < R
__global__ void sum_rows_kernel(const float* __restrict__ part, int ld, float* __restrict__ out, int n, int R) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float s = 0.f;
  for (int j = 0; j < n; j++) s += part[(size_t)j * ld + r];
  out[r] += s;
}

// ------------------------------------------------------------------------------------------------
// aux up-sampling + layout change (wavenet.py:124-154)
// ------------------------------------------------------------------------------------------------
__global__ void aux_upsample_fwd_kernel(const float* __restrict__ h, const float* __restrict__ w,
                                        const float* __restrict__ bias, float* __restrict__ haux, int B, int A,
                                        int Ap, int Tf, int U) {
  const int T = (U > 0) ? Tf * U : Tf;
  const int64_t total = (int64_t)B * T * Ap;
  const float bv = (U > 0) ? bias[0] : 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / Ap;
    const int a = (int)(i - bt * Ap);
    const int b = (int)(bt / T);
    const int t = (int)(bt - (int64_t)b * T);
    float v = 0.f;
    if (a < A) {
      if (U > 0) {
        const int tf = t / U, j = t - tf * U;
        v = fmaf(__ldg(h + ((size_t)b * A + a) * Tf + tf), __ldg(w + j), bv);
      } else {
        v = __ldg(h + ((size_t)b * A + a) * Tf + t);
      }
    }
    haux[i] = v;
  }
}

// Ap % 4 == 0: one thread per 4 aux channels of a row, 16-byte stores
__global__ void __launch_bounds__(256) aux_upsample_fwd_v4_kernel(const float* __restrict__ h, const float* __restrict__ w,
                                                                  const float* __restrict__ bias, float4* __restrict__ haux,
                                                                  int B, int A, int Ap4, int Tf, int U) {
  const int T = (U > 0) ? Tf * U : Tf;
  const int64_t total = (int64_t)B * T * Ap4;
  const float bv = (U > 0) ? bias[0] : 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / Ap4;
    const int a0 = (int)(i - bt * Ap4) * 4;
    const int b = (int)(bt / T);
    const int t = (int)(bt - (int64_t)b * T);
    const int tf = (U > 0) ? t / U : t;
    const float wj = (U > 0) ? __ldg(w + (t - tf * U)) : 1.f;
    float v[4];
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int a = a0 + c;
      v[c] = (a < A) ? ((U > 0) ? fmaf(__ldg(h + ((size_t)b * A + a) * Tf + tf), wj, bv)
                                : __ldg(h + ((size_t)b * A + a) * Tf + tf))
                     : 0.f;
    }
    haux[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// dw[j] += sum_{b,a,tf} h[b][a][tf] * dhaux[b][tf*U+j][a] ; dbias += sum_{b,t,a<A} dhaux
// block = one (b, tf); warp-strided over j, lanes over a.
__global__ void aux_upsample_bwd_kernel(const float* __restrict__ h, const float* __restrict__ dhaux,
                                        float* __restrict__ part, int B, int A, int Ap, int Tf, int U) {
  // Warp w of a block owns the sub-sample offsets j = w, w + nwarps, ... and keeps their partial sums in REGISTERS over
  // all the (b, tf) items of the block (lanes = aux channels); the block writes its partials part[block][0 .. U-1] (dw)
  // and part[block][U] (dbias), which sum_rows_kernel adds up in block order (no atomics: the result does not depend on
  // scheduling).
  constexpr int kMaxJ = 16;                                   // j values per warp and pass (128 per pass with 8 warps)
  constexpr int kAC = 8;                                      // aux channels per lane: A <= 256
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ float sb[32];
  float btot = 0.f;
  for (int jbase = 0; jbase < U; jbase += kMaxJ * nwarps) {   // (one pass for U <= 128; 256 = ljspeech-melspc: two)
    float acc[kMaxJ];
#pragma unroll
    for (int i = 0; i < kMaxJ; i++) acc[i] = 0.f;
    for (int64_t item = blockIdx.x; item < (int64_t)B * Tf; item += gridDim.x) {
      const int b = (int)(item / Tf), tf = (int)(item % Tf);
      float hv[kAC];                                          // h[b][a][tf] for a = lane, lane + 32, ...
#pragma unroll
      for (int c = 0; c < kAC; c++) {
        const int a = lane + 32 * c;
        hv[c] = (a < A) ? __ldg(h + ((size_t)b * A + a) * Tf + tf) : 0.f;
      }
      const float* base = dhaux + ((size_t)b * Tf * U + (size_t)tf * U) * Ap;
#pragma unroll
      for (int i = 0; i < kMaxJ; i++) {
        const int j = jbase + warp + i * nwarps;
        if (j < U) {
          const float* row = base + (size_t)j * Ap;
#pragma unroll
          for (int c = 0; c < kAC; c++) {
            const int a = lane + 32 * c;
            if (a < A) {
              const float g = __ldg(row + a);
              acc[i] = fmaf(g, hv[c], acc[i]);
              btot += g;
            }
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxJ; i++) {
      const int j = jbase + warp + i * nwarps;
      const float v = warp_sum(acc[i]);
      if (j < U && lane == 0) part[(size_t)blockIdx.x * (U + 1) + j] = v;
    }
  }
  btot = warp_sum(btot);
  if (lane == 0) sb[warp] = btot;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < nwarps; i++) s += sb[i];
    part[(size_t)blockIdx.x * (U + 1) + U] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// cross entropy (mean over B*(T-start) rows) + gradient; one warp per (b,t) row of Q logits
// ------------------------------------------------------------------------------------------------
// dlogits may alias logits (in-place: the fused training entry never keeps the logits): every lane finishes reading
// a row -- including the target logit -- before any lane overwrites it.
__global__ void cross_entropy_kernel(const float* logits, const int64_t* __restrict__ target,
                                     double* __restrict__ loss_part, float* dlogits, int B, int T, int Q,
                                     int start, float inv_n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t nrows = (int64_t)B * T;
  double local = 0.0;
  for (int64_t row = (int64_t)blockIdx.x * nwarps + warp; row < nrows; row += (int64_t)gridDim.x * nwarps) {
    const int t = (int)(row % T);
    const float* lg = logits + row * Q;
    float* dl = dlogits ? dlogits + row * Q : nullptr;
    if (t < start) {
      if (dl)
        for (int q = lane; q < Q; q += 32) dl[q] = 0.f;
      continue;
    }
    float m = -INFINITY;
    for (int q = lane; q < Q; q += 32) m = fmaxf(m, lg[q]);
    m = warp_max(m);
    float s = 0.f;
    for (int q = lane; q < Q; q += 32) s += expf(lg[q] - m);
    s = warp_sum(s);
    const float lse = m + logf(s);
    int64_t tg = target[row];
    if (tg < 0 || tg >= Q) {   // torch's CrossEntropyLoss asserts here; flag it loudly instead of reading out of bounds
      if (lane == 0) local += (double)NAN;
      tg = 0;
    }
    const float ltg = lg[tg];
    if (lane == 0) local += (double)(lse - ltg);
    if (dl) {
      const float inv_s = 1.0f / s;
      __syncwarp();
      for (int q = lane; q < Q; q += 32) {
        float p = expf(lg[q] - m) * inv_s;
        if (q == tg) p -= 1.0f;
        dl[q] = p * inv_n;
      }
    }
  }
  __shared__ double sl[32];
  if (lane == 0) sl[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < nwarps; i++) s += sl[i];
    loss_part[blockIdx.x] = s * (double)inv_n;   // summed in block order by sum_loss_kernel
  }
}

// Q == 256 fast path: the row lives in registers (two 16-byte loads per lane), one pass for max / exp / sum, two 16-byte
// stores for the gradient -- instead of three passes of 4-byte loads over the row.
__global__ void __launch_bounds__(256) cross_entropy_q256_kernel(const float* logits, const int64_t* __restrict__ target,
                                                                 double* __restrict__ loss_part, float* dlogits, int B, int T,
                                                                 int start, float inv_n) {
  constexpr int Q = 256;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t nrows = (int64_t)B * T;
  double local = 0.0;
  for (int64_t row = (int64_t)blockIdx.x * nwarps + warp; row < nrows; row += (int64_t)gridDim.x * nwarps) {
    const int t = (int)(row % T);
    const float4* lg4 = reinterpret_cast<const float4*>(logits + row * Q);
    float4* dl4 = dlogits ? reinterpret_cast<float4*>(dlogits + row * Q) : nullptr;
    if (t < start) {
      if (dl4) { dl4[lane] = make_float4(0.f, 0.f, 0.f, 0.f); dl4[32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f); }
      continue;
    }
    const float4 a = lg4[lane], b = lg4[32 + lane];     // columns 4*lane .. +3 and 128 + 4*lane .. +3
    float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    float m = v[0];
#pragma unroll
    for (int k = 1; k < 8; k++) m = fmaxf(m, v[k]);
    m = warp_max(m);
    float e[8], sum = 0.f;
#pragma unroll
    for (int k = 0; k < 8; k++) { e[k] = expf(v[k] - m); sum += e[k]; }
    sum = warp_sum(sum);
    const float lse = m + logf(sum);
    int64_t tg = target[row];
    if (tg < 0 || tg >= Q) {
      if (lane == 0) local += (double)NAN;
      tg = 0;
    }
    const float ltg = logits[row * Q + tg];
    if (lane == 0) local += (double)(lse - ltg);
    if (dl4) {
      const float inv_s = 1.0f / sum;
      __syncwarp();
      float o[8];
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int q = (k < 4 ? 4 * lane + k : 128 + 4 * lane + (k - 4));
        float pr = e[k] * inv_s;
        if (q == (int)tg) pr -= 1.0f;
        o[k] = pr * inv_n;
      }
      dl4[lane] = make_float4(o[0], o[1], o[2], o[3]);
      dl4[32 + lane] = make_float4(o[4], o[5], o[6], o[7]);
    }
  }
  __shared__ double sl[32];
  if (lane == 0) sl[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < nwarps; i++) s += sl[i];
    loss_part[blockIdx.x] = s * (double)inv_n;   // summed in block order by sum_loss_kernel
  }
}

}  // namespace wnb

using namespace wnb;

// *loss_sum += part[0] + part[1] + ... + part[n-1], in that order
__global__ void sum_loss_kernel(const double* __restrict__ part, double* __restrict__ loss_sum, int n) {
  double s = 0.0;
  for (int i = 0; i < n; i++) s += part[i];
  *loss_sum += s;
}

extern "C" {

WNB_API int wnb_version(void) { return 100; }
WNB_API const char* wnb_last_error(void) { return wnb::g_err; }
WNB_API int64_t wnb_launch_count(void) { return wnb::g_launches.load(); }

WNB_API int wnb_profile_enable(int on) {
  using namespace wnb;
  for (auto& r : g_prof_recs) { g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1); }
  g_prof_recs.clear();
  g_prof_on = on != 0;
  return WNB_OK;
}

WNB_API int wnb_profile_read(int kind, double* total_ms, int* launches) {
  using namespace wnb;
  WNB_REQUIRE(total_ms && launches && kind >= 0 && kind < WNB_PROF_KINDS, "profile_read: bad arguments");
  double tot = 0.0;
  int n = 0;
  for (auto& r : g_prof_recs) {
    if (r.kind != kind) continue;
    WNB_CUDA(cudaEventSynchronize(r.e1));
    float ms = 0.f;
    WNB_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
    tot += ms;
    n++;
  }
  *total_ms = tot;
  *launches = n;
  return WNB_OK;
}

WNB_API int wnb_mulaw_encode_f32(const float* x, int64_t* y, int64_t n, int mu, void* stream) {
  WNB_REQUIRE(n >= 0 && mu >= 2, "mulaw_encode_f32: bad n/mu");
  if (n == 0) return WNB_OK;
  const float m = (float)(mu - 1);
  mulaw_encode_f32_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n, m,
                                                                             log(1.0 + (double)(mu - 1)));
  WNB_CHECK_LAUNCH("mulaw_encode_f32");
  return WNB_OK;
}

WNB_API int wnb_mulaw_encode_f64(const double* x, int64_t* y, int64_t n, int mu, void* stream) {
  WNB_REQUIRE(n >= 0 && mu >= 2, "mulaw_encode_f64: bad n/mu");
  if (n == 0) return WNB_OK;
  mulaw_encode_f64_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n, (double)(mu - 1),
                                                                             log(1.0 + (double)(mu - 1)));
  WNB_CHECK_LAUNCH("mulaw_encode_f64");
  return WNB_OK;
}

WNB_API int wnb_mulaw_decode_f64(const int64_t* y, double* x, int64_t n, int mu, void* stream) {
  WNB_REQUIRE(n >= 0 && mu >= 2, "mulaw_decode_f64: bad n/mu");
  if (n == 0) return WNB_OK;
  MulawTable tab;
  const double m = (double)(mu - 1);
  for (int q = 0; q < 256; q++) {
    volatile double fx = ((double)q - 0.5) / m * 2.0 - 1.0;
    const double sgn = (fx > 0.) ? 1. : ((fx < 0.) ? -1. : 0.);
    volatile double pw = pow(1.0 + m, fabs(fx));
    tab.v[q] = sgn / m * (pw - 1.0);
  }
  mulaw_decode_f64_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(y, x, n, m, mu, tab);
  WNB_CHECK_LAUNCH("mulaw_decode_f64");
  return WNB_OK;
}

WNB_API int wnb_lut_i16(const int32_t* idx, const int16_t* table, int16_t* out, int64_t n, int ntab, void* stream) {
  WNB_REQUIRE(n >= 0 && ntab > 0 && (n == 0 || (idx && table && out)), "lut_i16: bad arguments");
  if (n == 0) return WNB_OK;
  lut_i16_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(idx, table, out, n, ntab);
  WNB_CHECK_LAUNCH("lut_i16");
  return WNB_OK;
}

WNB_API int wnb_front_embed_fwd(const int64_t* x, const float* wf, const float* bias, float* out, int B, int T, int Q,
                        int R, int ks, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && Q > 0 && R > 0 && ks >= 1, "front_embed_fwd: bad shape");
  const bool v4 = R % 4 == 0 && 256 % (R / 4) == 0 &&
                  ((reinterpret_cast<uintptr_t>(wf) | reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  if (v4) {
    const int rows_per_blk = 256 / (R / 4);
    front_embed_fwd_v4_kernel<<<grid_for(cdiv64((int64_t)B * T, rows_per_blk) * 256, 256), 256, 0, (cudaStream_t)stream>>>(
        x, reinterpret_cast<const float4*>(wf), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(out), B, T,
        Q, R / 4, ks);
  } else {
    front_embed_fwd_kernel<<<grid_for((int64_t)B * T * R, 256), 256, 0, (cudaStream_t)stream>>>(x, wf, bias, out, B, T,
                                                                                                Q, R, ks);
  }
  WNB_CHECK_LAUNCH("front_embed_fwd");
  return WNB_OK;
}

WNB_API int wnb_front_embed_bwd(const int64_t* x, const float* dout, float* dwf, float* dbias, int B, int T, int Q, int R,
                        int ks, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && Q > 0 && R > 0 && ks >= 1, "front_embed_bwd: bad shape");
  WNB_REQUIRE(ks <= 4, "front_embed_bwd: kernel_size <= 4 (got %d)", ks);
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = R % 4 == 0 && R / 4 <= 512 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0;
  WNB_REQUIRE(v4 || R <= 512, "front_embed_bwd: n_resch <= 512 unless it is a multiple of 4 (got %d)", R);
  const int64_t nrows = (int64_t)B * T;
  float* qpart = static_cast<float*>(scratch_buffer(st, SCRATCH_EMBED, ((size_t)Q * R + nrows) * sizeof(float)));
  WNB_REQUIRE(qpart, "front_embed_bwd: cannot allocate the scratch buffer");
  int* tok = reinterpret_cast<int*>(qpart + (size_t)Q * R);
  token_kernel<<<grid_for(nrows, 256), 256, 0, st>>>(x, tok, nrows, Q);
  WNB_CHECK_LAUNCH("front_embed_bwd_tokens");
  const size_t tab_bytes = (size_t)ks * Q * R * sizeof(float);
  if (v4 && 256 % (R / 4) == 0 && tab_bytes <= 160 * 1024) {
    // chunked tables in shared memory: one chunk per SM
    const int nchunks = device_sms();
    const int64_t chunk = (nrows + nchunks - 1) / nchunks;
    float* part = static_cast<float*>(scratch_buffer(st, SCRATCH_EMBED_PART, (size_t)nchunks * tab_bytes));
    WNB_REQUIRE(part, "front_embed_bwd: cannot allocate the scratch buffer");
    WNB_CUDA(ensure_dynamic_smem(reinterpret_cast<const void*>(front_embed_bwd_chunk_kernel), tab_bytes));
    front_embed_bwd_chunk_kernel<<<nchunks, 256, tab_bytes, st>>>(tok, reinterpret_cast<const float4*>(dout), part, B, T, Q,
                                                                  R / 4, ks, chunk);
    WNB_CHECK_LAUNCH("front_embed_bwd_chunk");
    const int n = ks * Q * R;
    front_embed_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(part, dwf, qpart, nchunks, n, (ks - 1) * Q * R);
    WNB_CHECK_LAUNCH("front_embed_bwd_reduce");
  } else if (v4) {
    const int Rv = R / 4;
    front_embed_bwd_kernel<4><<<Q, (512 / Rv) * Rv, 0, st>>>(tok, dout, dwf, qpart, B, T, Q, Rv, ks);
  } else {
    front_embed_bwd_kernel<1><<<Q, (512 / R) * R, 0, st>>>(tok, dout, dwf, qpart, B, T, Q, R, ks);
  }
  WNB_CHECK_LAUNCH("front_embed_bwd");
  sum_rows_kernel<<<(R + 127) / 128, 128, 0, st>>>(qpart, R, dbias, Q, R);
  WNB_CHECK_LAUNCH("front_embed_bwd_bias");
  return WNB_OK;
}

WNB_API int wnb_aux_upsample_fwd(const float* h, const float* w, const float* bias, float* haux, int B, int A, int Ap,
                         int Tf, int U, void* stream) {
  WNB_REQUIRE(B > 0 && A > 0 && Ap >= A && Tf > 0 && U >= 0, "aux_upsample_fwd: bad shape");
  WNB_REQUIRE(U == 0 || (w && bias), "aux_upsample_fwd: U>0 needs w and bias");
  const int64_t T = U > 0 ? (int64_t)Tf * U : Tf;
  if (Ap % 4 == 0 && (reinterpret_cast<uintptr_t>(haux) & 15) == 0)
    aux_upsample_fwd_v4_kernel<<<grid_for((int64_t)B * T * (Ap / 4), 256), 256, 0, (cudaStream_t)stream>>>(
        h, w, bias, reinterpret_cast<float4*>(haux), B, A, Ap / 4, Tf, U);
  else
    aux_upsample_fwd_kernel<<<grid_for((int64_t)B * T * Ap, 256), 256, 0, (cudaStream_t)stream>>>(h, w, bias, haux, B,
                                                                                                  A, Ap, Tf, U);
  WNB_CHECK_LAUNCH("aux_upsample_fwd");
  return WNB_OK;
}

WNB_API int wnb_aux_upsample_bwd(const float* h, const float* dhaux, float* dw, float* dbias, int B, int A, int Ap, int Tf,
                         int U, void* stream) {
  WNB_REQUIRE(B > 0 && A > 0 && Ap >= A && Tf > 0 && U > 0, "aux_upsample_bwd: bad shape");
  WNB_REQUIRE(A <= 256, "aux_upsample_bwd: n_aux <= 256 (got %d)", A);
  int64_t items = (int64_t)B * Tf;
  int grid = (int)(items < device_sms() * 4 ? items : device_sms() * 4);
  cudaStream_t st = (cudaStream_t)stream;
  float* part = static_cast<float*>(scratch_buffer(st, SCRATCH_AUX, (size_t)grid * (U + 1) * sizeof(float)));
  WNB_REQUIRE(part, "aux_upsample_bwd: cannot allocate the scratch buffer");
  aux_upsample_bwd_kernel<<<grid, 256, 0, st>>>(h, dhaux, part, B, A, Ap, Tf, U);
  WNB_CHECK_LAUNCH("aux_upsample_bwd");
  // dw: columns 0 .. U-1 of the partials, dbias: column U
  sum_rows_kernel<<<(U + 127) / 128, 128, 0, st>>>(part, U + 1, dw, grid, U);
  WNB_CHECK_LAUNCH("aux_upsample_bwd_w");
  sum_rows_kernel<<<1, 32, 0, st>>>(part + U, U + 1, dbias, grid, 1);
  WNB_CHECK_LAUNCH("aux_upsample_bwd_b");
  return WNB_OK;
}

WNB_API int wnb_cross_entropy(const float* logits, const int64_t* target, double* loss_sum, float* dlogits, int B, int T,
                      int Q, int start, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && Q > 0 && start >= 0 && start < T, "cross_entropy: bad shape (start=%d T=%d)", start,
              T);
  const int64_t n = (int64_t)B * (T - start);
  const int64_t nrows = (int64_t)B * T;
  int grid = (int)(cdiv64(nrows, 8) < device_sms() * 8 ? cdiv64(nrows, 8) : device_sms() * 8);
  cudaStream_t st = (cudaStream_t)stream;
  double* part = static_cast<double*>(scratch_buffer(st, SCRATCH_LOSS, (size_t)grid * sizeof(double)));
  WNB_REQUIRE(part, "cross_entropy: cannot allocate the scratch buffer");
  if (Q == 256 && ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(dlogits)) & 15) == 0)
    cross_entropy_q256_kernel<<<grid, 256, 0, st>>>(logits, target, part, dlogits, B, T, start, 1.0f / (float)n);
  else
    cross_entropy_kernel<<<grid, 256, 0, st>>>(logits, target, part, dlogits, B, T, Q, start, 1.0f / (float)n);
  WNB_CHECK_LAUNCH("cross_entropy");
  sum_loss_kernel<<<1, 1, 0, st>>>(part, loss_sum, grid);
  WNB_CHECK_LAUNCH("cross_entropy_sum");
  return WNB_OK;
}

}  // extern "C"
