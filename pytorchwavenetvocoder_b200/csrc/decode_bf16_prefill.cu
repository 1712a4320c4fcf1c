// decode_bf16_prefill.cu -- the teacher-forced warm-up of the bf16 decoder (padded positions 0 .. P - 2), computed in
// parallel over time and bit-identical to the sequential warm-up of decode_bf16_kernel.
//
// What the free-running steps need from the warm-up is only the dilation queues: layer l's ring holds bf16(x_l(t)) for
// t in [P - 1 - (ks - 1) d_l, P - 2].  Every x_l(t) with t < P - 1 depends only on the seed prefix, the aux features and
// the weights, so per layer all warm-up positions are independent, like the utterances of a batch.  Layer l's input is
// needed on its pruned window only, the last S_l = (ks - 1) (d_l + ... + d_{L-1}) positions before P - 1
// (wnb_decode_prefill_windows), so the cost does not depend on the seed length.
//
// Bit identity.  decode_bf16_kernel sums each product inside wgmma, in an order and at a precision PTX does not specify,
// so no SIMT code restates it.  The prefill issues the same instructions on the same operands in the same K order: the
// M = 64 rows of a product are 64 consecutive positions of one utterance here, 64 utterances there.  An output element
// (m, n) of wgmma depends on row m of A, column n of B and its accumulator only, so the row's meaning does not matter.
//   * weights: CTA r of the decoder's cluster owns output slice r; here slice r of a tile reads the same packed per-CTA
//     stream (nets/wavenet.py::_decode_bf16_pack), gate and res chunks and their fp32 bias tails;
//   * products: product<NG> for the gate over K = [aux (Ak/64 chunks) | taps j = 0 .. ks-2, tap j = x_l(t - (ks-1-j) d),
//     R/64 chunks each | x_l(t) (R/64)], product<NR> (NR = R/8 + S/8) for res+skip over K = z; the skip columns are
//     computed and dropped, so the instruction shape stays the decoder's; A fragments through mma_tile
//     (decode_bf16_common.cuh), accumulators zeroed first;
//   * rounding points, as the decoder's step: x_0 = bf + wf[0][q_0] + wf[1][q_1] (+ wf[2][q_2]) in fp32; the aux column
//     fmaf(h, up_w[j % U], up_b) (h itself when U = 0) then cvt.rn.bf16x2; z = sigmoidf_(g + b1) * tanhf(g' + b1') then
//     bf16; x_{l+1} = x_l + (d + b2) in fp32; the A operands and the queues hold bf16(x_l); taps at positions < 0 are zero.
//
// Work split: one launch for the front (x_0 on its window), then per layer l < L - 1 two launches over (tile of 64
// positions, slice r = 0..7).  The gate launch writes slice r's channels of z as bf16 to scratch; the res launch reads
// all R channels of z, updates slice r's channels of x in place (fp32 and bf16 copies) and writes the queue of layer
// l + 1.  No cluster is needed: the z exchange goes through global memory and the launch boundary.  One fp32 and one bf16
// copy of x are enough: a res launch reads and writes x_l(t) only for its own positions and channels, and the gate
// launch that read bf16(x_l) has finished.  Inside a CTA a producer warp streams the weight chunks through a ring of
// shared-memory stages with cp.async.bulk (the decoder's Ring), and the consumer warpgroup double-buffers the A tiles
// with cp.async (16-byte units into the 128B swizzle, zero-filled past the window).
//
// Queues: the decoder's layout (per cluster of ceil(B / ncl) utterances, per layer, (ks - 1) d_l slots of R/64 swizzled
// [64 rows][64] bf16 tiles; position t in slot t mod (ks - 1) d_l).  A row m >= nu of a cluster holds the values of its
// last utterance, because the decoder computes those rows from min(row, nu - 1); the prefill writes them too, so the
// whole workspace compares equal.
//
// Every mbarrier wait is bounded by %globaltimer (tc_ptx.cuh) and traps; nothing in the wgmma pipeline makes a call.
#include "decode_bf16_common.cuh"

namespace wnb {
namespace dbp {

using db::kCL;
using db::kCons;
using db::kM;
using db::kQ;
using db::kTile;

constexpr int kMaxL = 64;
constexpr int kThreads = kCons + 32;      // consumer warpgroup + producer warp
constexpr int kMaxStages = 4;
constexpr int kSmemBudget = 112 * 1024;   // dynamic shared memory of one CTA: two CTAs per SM

struct Params {
  const int32_t* xs;              // (B, P) seed prefix
  const float* h; const float* up_w; const float* up_b; const float* wf; const float* bf;
  const unsigned char* weights;   // the decoder's 8 per-CTA streams
  unsigned char* queues;
  float* xf;                      // x_l fp32, [B][nw][R]: position t at row t - base
  uint16_t* xb;                   // bf16(x_l), same layout
  uint16_t* zb;                   // z of the current layer, bf16, same layout
  int B, P, n_pad, Th, A, Ak, U, L, ks, nstage, stage_bytes, bc;
  int base, nw;
  long long cta_bytes, layer_bytes, gate_bytes, q_cluster;
  int dil[kMaxL];
  long long qslot[kMaxL];         // first slot of layer l's queue
  int lo[kMaxL];                  // first position of layer l's input window: max(0, P - 1 - S_l)
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// A tile of 64 rows, row m = position t_first + m, channels ch0 .. ch0 + 63 of a [nw][R] bf16 array (row t - base), into
// the swizzled tile at `dst`; rows outside [max(base, 0), last] read as zero.  One commit group per thread.
template <int R>
__device__ __forceinline__ void load_rows(uint32_t dst, const uint16_t* src, int t_first, int ch0, int base, int last,
                                          int tid) {
#pragma unroll
  for (int u = tid; u < kM * 8; u += kCons) {
    const int row = u >> 3, un = u & 7, t = t_first + row;
    const bool ok = t >= base && t <= last;
    cp_async16(dst + db::tile_off(row, 8 * un), ok ? src + (size_t)(t - base) * R + ch0 + 8 * un : src, ok ? 16u : 0u);
  }
  cp_async_commit();
}

// bf16 pair v of channels ch, ch + 1 of x_l(t) of utterance b into layer l's queue, if t is one of its last positions;
// the last utterance of a cluster fills the padding rows as well
template <int R>
__device__ __forceinline__ void put_queue(const Params& p, int l, int b, int t, int ch, uint32_t v) {
  const int qlen = (p.ks - 1) * p.dil[l];
  if (t < p.P - 1 - qlen) return;
  const int cl = b / p.bc, row = b - cl * p.bc, nu = min(p.bc, p.B - cl * p.bc);
  unsigned char* q = p.queues + (size_t)cl * p.q_cluster + (size_t)(p.qslot[l] + t % qlen) * (R / 64) * kTile;
  const int end = row == nu - 1 ? kM : row + 1;
  for (int m = row; m < end; m++) *reinterpret_cast<uint32_t*>(q + db::act_off(m, ch)) = v;
}

// x_0(t) for t in [lo[0], P - 2], channel pairs: the decoder's step prologue, in its order
template <int R>
__global__ void prefill_front_kernel(const Params p) {
  const int n = p.P - 1 - p.lo[0], ks = p.ks;
  const long long total = (long long)p.B * n * (R / 2);
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = 2 * (int)(e % (R / 2));
    const long long bt = e / (R / 2);
    const int t = p.lo[0] + (int)(bt % n), b = (int)(bt / n);
    float v[2] = {__ldg(p.bf + c), __ldg(p.bf + c + 1)};
    for (int k = 0; k < ks; k++) {
      const int pp = t - (ks - 1 - k);
      if (pp < 0) continue;
      int q = p.xs[(size_t)b * p.P + pp];
      q %= kQ;
      if (q < 0) q += kQ;
      const float* w = p.wf + ((size_t)k * kQ + q) * R + c;
      v[0] += __ldg(w);
      v[1] += __ldg(w + 1);
    }
    const size_t at = ((size_t)b * p.nw + (t - p.base)) * R + c;
    *reinterpret_cast<float2*>(p.xf + at) = make_float2(v[0], v[1]);
    const uint32_t vb = ptx::cvt_bf16x2(v[0], v[1]);
    *reinterpret_cast<uint32_t*>(p.xb + at) = vb;
    put_queue<R>(p, 0, b, t, c, vb);
  }
}

// the CTA's tile (64 positions t0 .. of utterance b, output slice r) of layer l's launches, which compute x_{l+1} on
// [lo[l + 1], P - 2]; shared-memory carve-up: ring (1024-byte aligned), two A tiles, the aux tiles (gate only)
struct Tile {
  int r, b, t0, last;
  uint32_t ring, a, aux;
  __device__ __forceinline__ Tile(const Params& p, int l, unsigned char* smem_raw) {
    r = blockIdx.x % kCL;
    last = p.P - 2;
    const int lo = p.lo[l + 1], per = (last - lo) / kM + 1, tile = blockIdx.x / kCL;
    b = tile / per;
    t0 = lo + (tile - b * per) * kM;
    const uint32_t raw = ptx::smem_u32(smem_raw);
    ring = (raw + 1023u) & ~1023u;
    a = ring + (uint32_t)(p.nstage * p.stage_bytes);
    aux = a + 2 * kTile;
  }
};

// producer warp: nch chunks of the CTA's stream from w, every chunk n_rows x 64 bf16, the last one with its bias tail
__device__ __forceinline__ void produce(const Params& p, const unsigned char* w, int nch, int n_rows, uint32_t ring,
                                        uint64_t* full, uint64_t* empty) {
  int st = 0;
  uint32_t ph = 0;
  for (int c = 0; c < nch; c++) {
    const uint32_t bytes = n_rows * 128 + (c == nch - 1 ? n_rows * 4 : 0);
    ptx::mbar_wait(&empty[st], ph ^ 1u);
    ptx::mbar_arrive_expect_tx(&full[st], bytes);
    db::bulk_g2s(ring + (uint32_t)(st * p.stage_bytes), w, bytes, &full[st]);
    w += bytes;
    if (++st == p.nstage) { st = 0; ph ^= 1u; }
  }
}

__device__ __forceinline__ void init_ring(const Params& p, uint64_t* full, uint64_t* empty) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstage; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kCons / 32);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
}

// gate of layer l: z = sigmoidf_(g + b1) * tanhf(g' + b1') of slice r's channels, bf16, to p.zb
template <int R>
__global__ void __launch_bounds__(kThreads, 2) prefill_gate_kernel(const Params p, int l) {
  constexpr int CR = R / kCL, NG = 2 * CR, KT = R / 64;
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[kMaxStages], empty[kMaxStages];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Tile T(p, l, smem_raw);
  const int nA = p.Ak / 64, ks = p.ks, d = p.dil[l], nch = nA + ks * KT;
  init_ring(p, full, empty);
  if (warp == kCons / 32) {
    if (lane == 0)
      produce(p, p.weights + (size_t)T.r * p.cta_bytes + (size_t)l * p.layer_bytes, nch, NG, T.ring, full, empty);
    return;
  }
  const int fr = 16 * warp + (lane >> 2), fk = 2 * (lane & 3);
  const uint16_t* xb = p.xb + (size_t)T.b * p.nw * R;
  // chunk c >= nA: k = c - nA, tap j = k / KT (j = ks - 1: x(t)) at rows t0 - (ks - 1 - j) d .., channels 64 (k % KT) ..
  auto load_a = [&](int c) {
    const int k = c - nA, j = k / KT;
    load_rows<R>(T.a + (uint32_t)((k & 1) * kTile), xb, T.t0 - (ks - 1 - j) * d, (k - j * KT) * 64, p.base, T.last, tid);
  };
  load_a(nA);
  // aux rows (bf16): the decoder's aux column at each row's position (rows past the window repeat the last one)
  for (int e = tid; e < kM * (p.Ak / 2); e += kCons) {
    const int row = e / (p.Ak / 2), a = 2 * (e - row * (p.Ak / 2));
    const int j = max(min(T.t0 + row, T.last) - p.n_pad, 0);
    float v[2];
#pragma unroll
    for (int t = 0; t < 2; t++) {
      v[t] = 0.f;
      if (a + t < p.A) {
        if (p.U > 0) {
          const int tf = min(j / p.U, p.Th - 1), jj = j % p.U;
          v[t] = fmaf(__ldg(p.h + ((size_t)T.b * p.A + a + t) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
        } else {
          v[t] = __ldg(p.h + ((size_t)T.b * p.A + a + t) * p.Th + min(j, p.Th - 1));
        }
      }
    }
    db::st_shared_b32(T.aux + db::act_off(row, a), ptx::cvt_bf16x2(v[0], v[1]));
  }
  db::cons_sync();
  db::Ring rg{T.ring, full, empty, p.nstage, p.stage_bytes, 0, 0u, -1};
  float g[NG / 2];
  const uint32_t last = db::product<NG>(
      g, rg, nch,
      [&](int c, uint32_t) -> uint32_t {
        return c < nA ? T.aux + (uint32_t)(c * kTile) : T.a + (uint32_t)(((c - nA) & 1) * kTile);
      },
      [&](int c) {
        if (c < nA) return;
        cp_async_wait_all();   // this chunk's A tile has landed, and every thread is done with chunk c - 1's
        db::cons_sync();
        if (c + 1 < nch) load_a(c + 1);
      },
      fr, fk, lane);
  const float* b1 = reinterpret_cast<const float*>(smem_raw + (last - ptx::smem_u32(smem_raw)) + NG * 128);
  uint16_t* zb = p.zb + (size_t)T.b * p.nw * R;
#pragma unroll
  for (int i = 0; i < CR / 2; i += 2) {
    const int row = fr + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + fk;
    float z[2];
#pragma unroll
    for (int e = 0; e < 2; e++) z[e] = sigmoidf_(g[i + e] + b1[col + e]) * tanhf(g[i + e + CR / 2] + b1[CR + col + e]);
    const int t = T.t0 + row;
    if (t <= T.last)
      *reinterpret_cast<uint32_t*>(zb + (size_t)(t - p.base) * R + T.r * CR + col) = ptx::cvt_bf16x2(z[0], z[1]);
  }
}

// res of layer l: x_{l+1} = x_l + (d + b2) on slice r's channels, in place, fp32 and bf16; layer l + 1's queue
template <int R, int S>
__global__ void __launch_bounds__(kThreads, 2) prefill_res_kernel(const Params p, int l) {
  constexpr int CR = R / kCL, CS = S / kCL, NR = CR + CS, KT = R / 64;
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[kMaxStages], empty[kMaxStages];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Tile T(p, l, smem_raw);
  init_ring(p, full, empty);
  if (warp == kCons / 32) {
    if (lane == 0)
      produce(p, p.weights + (size_t)T.r * p.cta_bytes + (size_t)l * p.layer_bytes + p.gate_bytes, KT, NR, T.ring,
              full, empty);
    return;
  }
  const int fr = 16 * warp + (lane >> 2), fk = 2 * (lane & 3);
  const uint16_t* zb = p.zb + (size_t)T.b * p.nw * R;
  auto load_z = [&](int c) { load_rows<R>(T.a + (uint32_t)((c & 1) * kTile), zb, T.t0, c * 64, p.base, T.last, tid); };
  load_z(0);
  db::Ring rg{T.ring, full, empty, p.nstage, p.stage_bytes, 0, 0u, -1};
  float d[NR / 2];
  const uint32_t last = db::product<NR>(
      d, rg, KT, [&](int c, uint32_t) -> uint32_t { return T.a + (uint32_t)((c & 1) * kTile); },
      [&](int c) {
        cp_async_wait_all();
        db::cons_sync();
        if (c + 1 < KT) load_z(c + 1);
      },
      fr, fk, lane);
  const float* b2 = reinterpret_cast<const float*>(smem_raw + (last - ptx::smem_u32(smem_raw)) + NR * 128);
#pragma unroll
  for (int i = 0; i < CR / 2; i += 2) {
    const int row = fr + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + fk;
    const int t = T.t0 + row;
    if (t > T.last) continue;
    const int ch = T.r * CR + col;
    const size_t at = ((size_t)T.b * p.nw + (t - p.base)) * R + ch;
    float2 x = *reinterpret_cast<const float2*>(p.xf + at);
    x.x += d[i] + b2[col];
    x.y += d[i + 1] + b2[col + 1];
    *reinterpret_cast<float2*>(p.xf + at) = x;
    const uint32_t vb = ptx::cvt_bf16x2(x.x, x.y);
    *reinterpret_cast<uint32_t*>(p.xb + at) = vb;
    put_queue<R>(p, l + 1, T.b, t, ch, vb);
  }
}

}  // namespace dbp

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static int dbp_stage_bytes(int R, int S) {
  const int NG = R / 4, NR = R / 8 + S / 8;
  const int b = (NG > NR ? NG : NR) * (128 + 4);   // the widest chunk with its bias tail
  return (b + 1023) / 1024 * 1024;
}
static size_t dbp_fixed_smem(int Ap) { return 1024 + (size_t)2 * db::kTile + (size_t)db_aux_k(Ap) / 64 * db::kTile; }

}  // namespace wnb

using namespace wnb;

extern "C" {

// fp32 and bf16 copies of x_l and bf16 z over the largest pruned window, min(S_0, P - 1) positions of B utterances
WNB_API size_t wnb_decode_bf16_prefill_workspace(int B, int P, int R, int ks, const int32_t* host_dilations, int L) {
  if (B <= 0 || P < 1 || R <= 0 || ks < 1 || L < 1 || L > dbp::kMaxL) return 0;
  int64_t S[dbp::kMaxL];
  if (wnb_decode_prefill_windows(host_dilations, L, ks, S) != WNB_OK) return 0;
  const int64_t nw = S[0] < P - 1 ? S[0] : P - 1;
  return (size_t)B * (size_t)nw * (size_t)R * (sizeof(float) + 2 * sizeof(uint16_t));
}

WNB_API int wnb_decode_bf16_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                    const float* wf, const float* bf, const void* weights,
                                    const int32_t* host_dilations, int L, void* queues, void* scratch, int B, int P,
                                    int n_pad, int Th, int A, int Ap, int R, int S, int ks, int U,
                                    void* stream_handle) {
  using namespace dbp;
  WNB_REQUIRE(B > 0 && P >= 1 && n_pad >= 0 && n_pad < P && Th >= 1 && A > 0 && Ap >= A && R > 0 && S > 0 && ks >= 1 &&
                  U >= 0 && L >= 1,
              "decode_bf16_prefill: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && weights && host_dilations && queues, "decode_bf16_prefill: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_bf16_prefill: U>0 needs upsampling weight and bias");
  if (!wnb_decode_bf16_supported(kQ, Ap, R, S, ks, L)) {
    set_error("decode_bf16_prefill: shape not covered (Ap %d, R %d, S %d, ks %d, L %d): see wnb_decode_bf16_supported",
              Ap, R, S, ks, L);
    return WNB_ERR_UNSUPPORTED;
  }
  Params p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf;
  p.weights = (const unsigned char*)weights; p.queues = (unsigned char*)queues;
  p.B = B; p.P = P; p.n_pad = n_pad; p.Th = Th; p.A = A; p.Ak = db_aux_k(Ap); p.U = U; p.L = L; p.ks = ks;
  int ncl;
  db_split(B, &ncl, &p.bc);
  long long slots = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1, "decode_bf16_prefill: dilations must be positive");
    p.dil[l] = host_dilations[l];
    p.qslot[l] = slots;
    slots += (long long)(ks - 1) * host_dilations[l];
  }
  p.q_cluster = slots * (long long)R * kM * 2;
  int64_t Sw[kMaxL];
  wnb_decode_prefill_windows(host_dilations, L, ks, Sw);
  for (int l = 0; l < L; l++) p.lo[l] = (int)(P - 1 - Sw[l] > 0 ? P - 1 - Sw[l] : 0);
  p.base = p.lo[0];
  p.nw = P - 1 - p.lo[0];
  WNB_REQUIRE(scratch || p.nw == 0, "decode_bf16_prefill: null scratch");
  const long long max_ctas = (long long)B * ((p.nw + kM - 1) / kM) * kCL;
  WNB_REQUIRE(max_ctas < 0x7fffffffLL, "decode_bf16_prefill: window too large");
  p.stage_bytes = dbp_stage_bytes(R, S);
  const size_t fixed = dbp_fixed_smem(Ap);
  p.nstage = (int)((kSmemBudget - (long long)fixed) / p.stage_bytes);
  if (p.nstage > kMaxStages) p.nstage = kMaxStages;
  WNB_REQUIRE(p.nstage >= 2, "decode_bf16_prefill: no weight ring fits");   // not reached for a covered shape
  p.layer_bytes = (long long)db_cta_bytes(Ap, R, S, ks);
  p.gate_bytes = (long long)db_gate_bytes(Ap, R, ks);
  p.cta_bytes = (long long)((size_t)L * db_cta_bytes(Ap, R, S, ks) + db_post_bytes(S));
  cudaStream_t st = (cudaStream_t)stream_handle;
  // queue slots of positions < 0 stay zero, as the sequential warm-up (which clears them first) leaves them
  WNB_CUDA(cudaMemsetAsync(queues, 0, (size_t)ncl * p.q_cluster, st));
  if (p.nw == 0) return WNB_OK;   // P == 1: no warm-up position
  const size_t xn = (size_t)B * p.nw * R;
  p.xf = (float*)scratch;
  p.xb = (uint16_t*)(p.xf + xn);
  p.zb = p.xb + xn;
  const size_t smem = fixed + (size_t)p.nstage * p.stage_bytes;
  auto run = [&](auto front, auto gate, auto res) -> int {
    {
      const long long total = (long long)B * p.nw * (R / 2);
      const int grid = (int)(total / 256 + 1 < 65536 ? total / 256 + 1 : 65536);
      front<<<grid, 256, 0, st>>>(p);
      WNB_CHECK_LAUNCH("decode_bf16_prefill");
    }
    WNB_CUDA(ensure_dynamic_smem((const void*)gate, smem));
    WNB_CUDA(ensure_dynamic_smem((const void*)res, smem));
    for (int l = 0; l + 1 < L; l++) {
      const int ctas = B * ((P - 1 - p.lo[l + 1] + kM - 1) / kM) * kCL;
      gate<<<ctas, kThreads, smem, st>>>(p, l);
      WNB_CHECK_LAUNCH("decode_bf16_prefill");
      res<<<ctas, kThreads, smem, st>>>(p, l);
      WNB_CHECK_LAUNCH("decode_bf16_prefill");
    }
    return WNB_OK;
  };
  if (R == 256) return run(prefill_front_kernel<256>, prefill_gate_kernel<256>, prefill_res_kernel<256, 256>);
  if (S == 256) return run(prefill_front_kernel<512>, prefill_gate_kernel<512>, prefill_res_kernel<512, 256>);
  return run(prefill_front_kernel<512>, prefill_gate_kernel<512>, prefill_res_kernel<512, 512>);
}

}  // extern "C"
