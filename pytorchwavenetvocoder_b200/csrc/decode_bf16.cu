// decode_bf16.cu -- opt-in bf16 tensor-core fast-generate kernel for the recipe-sized models (512 or 256 residual
// channels, 256 or 512 skip channels, kernel size 2 or 3): ONE 8-CTA THREAD-BLOCK CLUSTER PER <= 64 UTTERANCES.
//
// Why.  Above L2 size the fp32 decoders (decode_stream.cu, decode.cu) read every weight of the model on every step in
// every CTA, and one CTA carries 1 to 4 utterances.  Here the utterances of a batch are split evenly over ceil(B / 64)
// clusters; each cluster runs its utterances from the first to the last step on its own (no grid-wide barrier, clusters
// never talk to each other, so clusters that do not fit run in a later wave and nothing can deadlock).  Inside a
// cluster the utterances are the M = 64 rows of wgmma products (rows >= B_c compute garbage nobody reads), and CTA r
// owns 1/8 of every OUTPUT dimension, so each weight is read once per step per cluster, as bf16:
//   * gate channels [r R/8, (r+1) R/8), both the sigmoid and the tanh row; the residual channels of that same slice;
//     skip channels [r S/8, (r+1) S/8); post-1 outputs [r S/8, (r+1) S/8); classes [32 r, 32 r + 32).
//
// Products per layer (A = activations from registers, bf16; B = this CTA's weight slice, bf16, K-major, 128B-swizzled
// tiles of [N rows][64 k] that a producer warp streams through a ring of shared-memory stages with cp.async.bulk):
//   gate      N = 2 R/8   (R = 512: 128)   K = [aux (Ap rounded up to 64) | dilated taps (ks-1) R | x(t) R]
//   res+skip  N = R/8 + S/8 (512/256: 96)  K = R
//   post-1    N = S/8,  post-2  N = 32     K = S
// The W1 rows of a CTA are packed [R/8 sigmoid | R/8 tanh] of the same channels, so in the m64nN accumulator column c
// and its partner c + R/8 sit in the same thread (accumulator index i and i + R/16): the gate needs no exchange.  The
// fp32 residual slice and the running skip sum stay in registers in the res+skip accumulator layout for the whole step;
// the skip sum is added in layer order starting from the first block (python `0 + s0 + s1 ...`, like the fp32 decoders).
//
// Rounding points (the float64 emulation in tests/decode_bf16_reference.py restates them, and the layer-by-layer
// checker tests/decode_bf16_layers.py checks each stage against them from the queues): every weight except the
// front embedding is rounded to bf16 on the host (round to nearest even); the A operands of the products are bf16 of
// the fp32 values: aux, layer input x_l (both as the current column and as dilated taps), z, relu(skip sum) and
// relu(post-1).  Accumulation, biases, the residual stream, the skip sum, the gate (precise expf / tanhf) and the logits
// are fp32; the pick is the shared sampler of common.cuh on the fp32 logits.
//
// All-gathers inside the cluster.  Activation buffers are [C/64 tiles][64 rows][64 ch] bf16 with the 128B swizzle
// (16-byte unit u of row r stored at u ^ (r & 7)), so the A-fragment loads of a warp hit 32 distinct banks.  After its
// gate a CTA writes its z slice into its own z buffer, then sends it (st.async, 16 B per store, completing transaction
// bytes on the receiver's mbarrier) into the same place of the 7 peers; after its residual update it does the same with
// its x slice and the x buffers.  Two buffers are enough, because a peer can only write a CTA's buffer after that CTA has
// sent the data the peer's write depends on:
//   * a peer sends x_{l+1} only after its res product, which needs this CTA's z_l, sent after this CTA's gate -- the
//     only reader of x_l -- has finished;
//   * a peer sends z_{l+1} only after its gate of layer l+1, which needs this CTA's x_{l+1}, sent after this CTA's res
//     product -- the only reader of z_l -- has finished.
// The post network reuses them the same way: relu(skip) goes to the x buffers (read by post-1), relu(post-1) to the z
// buffers (read by post-2), and the 8 x 256 fp32 logits of utterance group g (rows 8g .. 8g+7) go to CTA g, into its aux
// buffer (free between the last gate of a step and the next step's aux).  CTA g's four warps pick their rows with
// sample_pick (common.cuh) and broadcast the picks into every CTA's pick history for the next step's front embedding.
// The same "cannot be one phase ahead" argument makes one mbarrier per buffer enough.
//
// The gate starts before x(t) arrives: its K segments run [aux | taps | x(t)], and the wait for the x all-gather sits
// in front of the first x(t) segment, so the tensor cores work through aux and taps while x is still in flight.
//
// Dilation queues (global memory, zeroed by the launcher): per cluster and layer l, (ks-1) d_l slots of the layer's
// input x_l as bf16, each slot R/64 swizzled [64 rows][64 ch] tiles (8 KB: one bulk copy).  The producer loads a tap tile
// into the same ring stage as the W1 chunk of the same K range.  CTA r writes its own channels of x_l(t) to slot
// t mod (ks-1) d_l in layer l's res epilogue.  Two hazards:
//   * write after read: that slot held x_l(t - (ks-1) d_l), the oldest tap of layer l at step t.  Every CTA's gate of
//     layer l (which consumed that tap: its TMA has completed) is over before any CTA gets past the z all-gather of
//     layer l, and the write comes after it.
//   * read after write (d = 1 taps are read one step after they are written): the write is a generic-proxy store, the
//     read a bulk copy in the async proxy, issued by another CTA's producer thread.  Each writer thread issues
//     fence.proxy.async.global after its queue stores; the consumer warpgroup then meets at a CTA barrier, and one thread
//     arrives with .release.cluster on the step barrier of every CTA of the cluster.  A producer waits on its step
//     barrier with .acquire.cluster for step t-1 before the first tap copy of step t.
// Taps before the start (t - s < 0) read slots nobody has written yet in this session: zeros.
//
// Warm-up: the teacher-forced prefix steps (P - 1 of them, P = max(T0, receptive field)) run the gate and res+skip
// products only (no post network, no pick); decode_bf16_prefill.cu computes the same queue bits in parallel over time,
// and a launch with pos0 = P - 1 continues from them.  Every wait is bounded by %globaltimer (tc_ptx.cuh) and traps;
// nothing in the wgmma pipeline makes a call.
//
// Shared memory per CTA (R = 512, ks = 3, A = 80 -> aux K 128): x 64 KB + z 64 KB + aux 16 KB + ring 3 x 24 KB
// (W1 chunk 128 x 64 bf16 = 16 KB + tap tile 8 KB) = 216 KB + 1 KB alignment slack + ~1.3 KB static, under the 227 KB
// limit; a fourth stage (240 KB) does not fit.  The launcher takes as many stages as fit, at most 8 (R = 256: 8).
#include "decode_bf16_common.cuh"

namespace wnb {
namespace db {

// kCL, kM (here: utterance rows per cluster), kQ, kQc, kTile, kCons: decode_bf16_common.cuh
constexpr int kMaxL = 64;
constexpr int kThreads = kCons + 32;      // + producer warp
constexpr int kMaxStages = 8;
constexpr int kSmemLimit = 227 * 1024;
constexpr int kStaticSmem = 2048;         // barriers, pick history, lengths (rounded up)

struct Params {
  int32_t* xs; const float* h; const float* up_w; const float* up_b; const float* wf; const float* bf;
  const unsigned char* weights;   // 8 per-CTA streams back to back (layout: wnb_decode_bf16_weights)
  unsigned char* queues;
  const int32_t* n_samples; const float* uniforms; float* logits_out;
  int B, P, max_n, n_pad, Th, A, Ak, U, mode, L, ks, nstage, stage_bytes, bc;
  int pos0, i0, i_last, h_last, stride_xs;   // the call's window (common.cuh DecodeWindow)
  long long cta_bytes;            // bytes of one CTA's stream
  long long q_cluster;            // bytes of one cluster's queues
  unsigned long long seed;
  int dil[kMaxL];
  long long qslot[kMaxL];         // first slot of layer l's queue
};

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_async_v4(uint32_t raddr, uint4 v, uint32_t rbar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(raddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async_v2(uint32_t raddr, uint32_t a, uint32_t b, uint32_t rbar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];"
               ::"r"(raddr), "r"(a), "r"(b), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async_b32(uint32_t raddr, uint32_t v, uint32_t rbar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
               ::"r"(raddr), "r"(v), "r"(rbar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// the step barrier: release.cluster arrive on CTA `rank`'s barrier at `bar`'s offset / acquire.cluster wait on our own
__device__ __forceinline__ void arrive_release_cluster(uint64_t* bar, uint32_t rank) {
  const uint32_t remote = mapa_u32(ptx::smem_u32(bar), rank);
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void wait_acquire_cluster(uint64_t* bar, uint32_t parity) {
  ptx::SpinGuard guard;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok) : "r"(ptx::smem_u32(bar)), "r"(parity) : "memory");
    if (ok) return;
    if (guard.expired()) __trap();
  }
}

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

template <int R, int S>
__global__ void __launch_bounds__(kThreads, 1) decode_bf16_kernel(const Params p) {
  constexpr int CR = R / kCL, CS = S / kCL;          // residual / skip channels per CTA
  constexpr int NG = 2 * CR, NR = CR + CS;            // gate and res+skip product widths
  constexpr int KT = R / 64;                          // 64-wide K tiles of R
  constexpr int KS = S / 64;
  static_assert(S <= R, "relu(skip) is gathered into the x buffers");
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[kMaxStages], empty[kMaxStages];
  __shared__ __align__(8) uint64_t xbar, zbar, lbar, pbar, qbar;
  __shared__ int32_t hist[4][kM];                     // picks by position (mod 4), every row of the cluster
  __shared__ int32_t s_n[kM];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t rank = cluster_ctarank();
  const int cl = blockIdx.x / kCL;
  const int u0 = cl * p.bc;
  const int nu = min(p.bc, p.B - u0);
  const int stride_xs = p.stride_xs;
  const int ks = p.ks, L = p.L;
  const int nA = p.Ak / 64, nT = (ks - 1) * KT;       // gate chunks: aux, taps, then KT of x(t)

  // carve-up: ring (1024-byte aligned: the swizzled B tiles), x, z, aux
  const uint32_t raw_u32 = ptx::smem_u32(smem_raw);
  const uint32_t ring_u32 = (raw_u32 + 1023u) & ~1023u;
  unsigned char* ring = smem_raw + (ring_u32 - raw_u32);
  unsigned char* xbuf = ring + (size_t)p.nstage * p.stage_bytes;
  unsigned char* zbuf = xbuf + KT * kTile;
  unsigned char* abuf = zbuf + KT * kTile;            // aux rows, and the logits of this CTA's utterance group
  const uint32_t x_u32 = ptx::smem_u32(xbuf), z_u32 = ptx::smem_u32(zbuf), a_u32 = ptx::smem_u32(abuf);

  if (tid == 0) {
    for (int i = 0; i < p.nstage; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kCons / 32);
    }
    ptx::mbar_init(&xbar, 1); ptx::mbar_init(&zbar, 1); ptx::mbar_init(&lbar, 1); ptx::mbar_init(&pbar, 1);
    ptx::mbar_init(&qbar, kCL);
    ptx::fence_barrier_init();
  }
  if (tid < kM) s_n[tid] = (tid < nu) ? p.i0 + p.n_samples[u0 + tid] : 0;   // absolute end
  __syncthreads();
  int nmax = 0;
  for (int u = 0; u < nu; u++) nmax = max(nmax, s_n[u]);
  if (nmax <= p.i0) return;   // (the same in every CTA of the cluster)
  // every CTA's barriers are initialised before the first remote arrival
  ptx::cluster_sync();
  const int last_pos = p.P - 1 + nmax - 1;
  const unsigned char* my_w = p.weights + (size_t)rank * p.cta_bytes;
  unsigned char* my_q = p.queues + (size_t)cl * p.q_cluster;

  if (warp == kCons / 32) {
    // ================================ producer warp ================================
    if (lane == 0) {
      int st = 0;
      uint32_t ph = 0, qph = 0;
      auto push = [&](const unsigned char* w, uint32_t wbytes, const unsigned char* tap) {
        ptx::mbar_wait(&empty[st], ph ^ 1u);
        ptx::mbar_arrive_expect_tx(&full[st], wbytes + (tap ? (uint32_t)kTile : 0u));
        const uint32_t dst = ring_u32 + (uint32_t)(st * p.stage_bytes);
        bulk_g2s(dst, w, wbytes, &full[st]);
        if (tap) bulk_g2s(dst + NG * 128, tap, kTile, &full[st]);
        if (++st == p.nstage) { st = 0; ph ^= 1u; }
      };
      for (int pos = p.pos0; pos <= last_pos; pos++) {
        const bool want = pos >= p.P - 1;
        const unsigned char* w = my_w;
        for (int l = 0; l < L; l++) {
          for (int c = 0; c < nA; c++, w += NG * 128) push(w, NG * 128, nullptr);
          if (l == 0 && pos > p.pos0) {
            // every CTA's queue writes of step pos-1 (and before) are visible to the async proxy (those of an earlier
            // launch are ordered by the launch boundary)
            wait_acquire_cluster(&qbar, qph);
            qph ^= 1u;
            fence_proxy_async_global();
          }
          const int d = p.dil[l], qlen = (ks - 1) * d;
          for (int j = 0; j < ks - 1; j++) {
            const int t = pos - (ks - 1 - j) * d;
            const int slot = ((t % qlen) + qlen) % qlen;
            const unsigned char* q = my_q + (size_t)(p.qslot[l] + slot) * KT * kTile;
            for (int c = 0; c < KT; c++, w += NG * 128) push(w, NG * 128, q + (size_t)c * kTile);
          }
          for (int c = 0; c < KT; c++) {
            const uint32_t b = NG * 128 + (c == KT - 1 ? NG * 4 : 0);
            push(w, b, nullptr);
            w += b;
          }
          for (int c = 0; c < KT; c++) {
            const uint32_t b = NR * 128 + (c == KT - 1 ? NR * 4 : 0);
            push(w, b, nullptr);
            w += b;
          }
        }
        if (want) {
          for (int c = 0; c < KS; c++) {
            const uint32_t b = CS * 128 + (c == KS - 1 ? CS * 4 : 0);
            push(w, b, nullptr);
            w += b;
          }
          for (int c = 0; c < KS; c++) {
            const uint32_t b = kQc * 128 + (c == KS - 1 ? kQc * 4 : 0);
            push(w, b, nullptr);
            w += b;
          }
        }
      }
    }
    __syncwarp();
    ptx::cluster_sync();      // no CTA leaves while a peer may still write its shared memory or arrive on its barriers
    return;
  }

  // ================================ consumer warpgroup ================================
  int fr = 16 * warp + (lane >> 2), fk = 2 * (lane & 3);   // fragment row (+ 8) and column pair (+ 8 j)
  // shared::cluster address deltas of the peers (rank + 1 .. rank + 7)
  uint32_t pdelta[kCL - 1];
#pragma unroll
  for (int i = 0; i < kCL - 1; i++) pdelta[i] = mapa_u32(x_u32, (rank + 1 + i) & (kCL - 1)) - x_u32;
  // send this CTA's slice (channels ch0 .. ch0 + nch of every row, already in its own buffer at `buf`) to the 7 peers
  auto send_slice = [&](uint32_t buf, int ch0, int nch, uint64_t* bar) {
    const int per_row = nch / 8, units = kM * per_row;
    const uint32_t lbar = ptx::smem_u32(bar);
    for (int u = tid; u < units; u += kCons) {
      const int row = u / per_row, c8 = ch0 + (u - row * per_row) * 8;
      const uint32_t a = buf + act_off(row, c8);
      uint4 v;
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
#pragma unroll
      for (int i = 0; i < kCL - 1; i++) st_async_v4(a + pdelta[i], v, lbar + pdelta[i]);
    }
  };
  auto expect = [&](uint64_t* bar, uint32_t bytes) {
    if (tid == 0) ptx::mbar_arrive_expect_tx(bar, bytes);
  };
  uint32_t xph = 0, zph = 0, lph = 0, pph = 0;
  auto wait_x = [&]() { ptx::mbar_wait(&xbar, xph); xph ^= 1u; };
  auto wait_z = [&]() { ptx::mbar_wait(&zbar, zph); zph ^= 1u; };
  auto no_pre = [](int) {};

  Ring rg{ring_u32, full, empty, p.nstage, p.stage_bytes, 0, 0u, -1};
  float xres[CR / 2];     // this CTA's residual channels, res+skip accumulator layout (index i < CR/2 of it)
  float skip[CS / 2];     // running skip sum (index CR/2 + i)
  auto row_of = [&](int i) { return fr + 8 * ((i >> 1) & 1); };
  auto col_of = [&](int i) { return 8 * (i >> 2) + fk + (i & 1); };

  for (int pos = p.pos0; pos <= last_pos; pos++) {
    const bool want = pos >= p.P - 1;
    const int istep = pos - (p.P - 1);
    // ---- step prologue: aux rows (bf16) and this CTA's slice of the front embedding (fp32, in registers) ----
    for (int e = tid; e < kM * (p.Ak / 2); e += kCons) {
      const int row = e / (p.Ak / 2), a = 2 * (e - row * (p.Ak / 2));
      const int ug = u0 + min(row, nu - 1);
      const int j = max(pos - p.n_pad, 0);
      float v[2];
#pragma unroll
      for (int t = 0; t < 2; t++) {
        v[t] = 0.f;
        if (a + t < p.A) {
          if (p.U > 0) {
            const int tf = min(j / p.U, p.h_last), jj = j % p.U;
            v[t] = fmaf(__ldg(p.h + ((size_t)ug * p.A + a + t) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
          } else {
            v[t] = __ldg(p.h + ((size_t)ug * p.A + a + t) * p.Th + min(j, p.h_last));
          }
        }
      }
      st_shared_b32(a_u32 + act_off(row, a), ptx::cvt_bf16x2(v[0], v[1]));
    }
    {
      int qk[2][3];
#pragma unroll
      for (int hh = 0; hh < 2; hh++) {
        const int row = fr + 8 * hh;
        const int ug = u0 + min(row, nu - 1);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const int pp = pos - (ks - 1 - k);
          int q = -1;
          if (k < ks && pp >= 0) {
            // the seed prefix and what earlier launches generated come from xs, this launch's picks from hist
            q = (pp < p.P || pp <= p.pos0) ? p.xs[(size_t)ug * stride_xs + pp] : hist[pp & 3][row];
            q %= kQ;
            if (q < 0) q += kQ;
          }
          qk[hh][k] = q;
        }
      }
      // v = bf + wf[0][q_0] + wf[1][q_1] (+ wf[2][q_2]), in that order; one k at a time keeps few loads in flight
      const float* bfc = p.bf + (int)rank * CR + fk;
#pragma unroll
      for (int i = 0; i < CR / 2; i++) xres[i] = __ldg(bfc + 8 * (i >> 2) + (i & 1));
#pragma unroll 1
      for (int k = 0; k < ks; k++) {
        const float* w0 = qk[0][k] >= 0 ? p.wf + ((size_t)k * kQ + qk[0][k]) * R + (int)rank * CR + fk : nullptr;
        const float* w1 = qk[1][k] >= 0 ? p.wf + ((size_t)k * kQ + qk[1][k]) * R + (int)rank * CR + fk : nullptr;
#pragma unroll
        for (int i = 0; i < CR / 2; i++) {
          const float* w = ((i >> 1) & 1) ? w1 : w0;
          if (w) xres[i] += __ldg(w + 8 * (i >> 2) + (i & 1));
        }
      }
#pragma unroll
      for (int i = 0; i < CR / 2; i += 2)
        st_shared_b32(x_u32 + act_off(row_of(i), (int)rank * CR + col_of(i)), ptx::cvt_bf16x2(xres[i], xres[i + 1]));
    }
    cons_sync();
    send_slice(x_u32, (int)rank * CR, CR, &xbar);
    expect(&xbar, (kCL - 1) * kM * CR * 2);

    for (int l = 0; l < L; l++) {
      fr = opaque(fr);
      fk = opaque(fk);
      rank = (uint32_t)opaque((int)rank);
      // ---------------- gate: [aux | taps | x(t)] ----------------
      float g[NG / 2];
      {
        const int first_x = nA + nT;
        const uint32_t last = product<NG>(
            g, rg, nA + nT + KT,
            [&](int c, uint32_t stage) -> uint32_t {
              return c < nA ? a_u32 + c * kTile : c < first_x ? stage + NG * 128 : x_u32 + (c - first_x) * kTile;
            },
            [&](int c) { if (c == first_x) wait_x(); }, fr, fk, lane);
        const float* b1 = reinterpret_cast<const float*>(ring + (last - ring_u32) + NG * 128);
#pragma unroll
        for (int i = 0; i < CR / 2; i += 2) {
          float z[2];
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int c = col_of(i + e);
            z[e] = sigmoidf_(g[i + e] + b1[c]) * tanhf(g[i + e + CR / 2] + b1[CR + c]);
          }
          st_shared_b32(z_u32 + act_off(row_of(i), (int)rank * CR + col_of(i)), ptx::cvt_bf16x2(z[0], z[1]));
        }
        rg.release(rg.prev, lane);
        rg.prev = -1;
      }
      cons_sync();
      send_slice(z_u32, (int)rank * CR, CR, &zbar);
      expect(&zbar, (kCL - 1) * kM * CR * 2);
      wait_z();
      // ---------------- res + skip ----------------
      {
        float d[NR / 2];
        const uint32_t last = product<NR>(
            d, rg, KT, [&](int c, uint32_t) -> uint32_t { return z_u32 + c * kTile; }, no_pre, fr, fk, lane);
        const float* b2 = reinterpret_cast<const float*>(ring + (last - ring_u32) + NR * 128);
        // x_l(pos) (this CTA's channels, bf16) -> slot pos mod (ks-1) d of layer l's queue: every CTA's gate of layer l
        // is over (they all sent z), so nobody still reads the tap this overwrites
        {
          const int qlen = (ks - 1) * p.dil[l];
          unsigned char* q = my_q + (size_t)(p.qslot[l] + pos % qlen) * KT * kTile;
#pragma unroll
          for (int i = 0; i < CR / 2; i += 2)
            *reinterpret_cast<uint32_t*>(q + act_off(row_of(i), (int)rank * CR + col_of(i))) =
                ptx::cvt_bf16x2(xres[i], xres[i + 1]);
        }
#pragma unroll
        for (int i = 0; i < CR / 2; i++) xres[i] += d[i] + b2[col_of(i)];
        if (want) {
#pragma unroll
          for (int i = 0; i < CS / 2; i++) {
            const float v = d[CR / 2 + i] + b2[col_of(CR / 2 + i)];
            skip[i] = (l == 0) ? v : skip[i] + v;
          }
        }
        rg.release(rg.prev, lane);
        rg.prev = -1;
      }
      if (l + 1 < L) {
#pragma unroll
        for (int i = 0; i < CR / 2; i += 2)
          st_shared_b32(x_u32 + act_off(row_of(i), (int)rank * CR + col_of(i)), ptx::cvt_bf16x2(xres[i], xres[i + 1]));
        cons_sync();
        send_slice(x_u32, (int)rank * CR, CR, &xbar);
        expect(&xbar, (kCL - 1) * kM * CR * 2);
      }
    }
    // ---- end of this step's queue writes: release them to every producer of the cluster ----
    fr = opaque(fr);
    fk = opaque(fk);
    rank = (uint32_t)opaque((int)rank);
    if (want) {
      // relu(skip sum) -> bf16 -> this CTA's channels of the x buffer (col_of(CR/2 + i) - CR = col_of(i))
#pragma unroll
      for (int i = 0; i < CS / 2; i += 2)
        st_shared_b32(x_u32 + act_off(row_of(i), (int)rank * CS + col_of(i)),
                      ptx::cvt_bf16x2(fmaxf(skip[i], 0.f), fmaxf(skip[i + 1], 0.f)));
    }
    fence_proxy_async_global();
    cons_sync();
    if (tid == 0)
      for (int r = 0; r < kCL; r++) arrive_release_cluster(&qbar, (uint32_t)r);
    if (!want) continue;

    // ---------------- post network ----------------
    send_slice(x_u32, (int)rank * CS, CS, &xbar);
    expect(&xbar, (kCL - 1) * kM * CS * 2);
    wait_x();
    {
      float d[CS / 2];
      const uint32_t last = product<CS>(
          d, rg, KS, [&](int c, uint32_t) -> uint32_t { return x_u32 + c * kTile; }, no_pre, fr, fk, lane);
      const float* bp1 = reinterpret_cast<const float*>(ring + (last - ring_u32) + CS * 128);
#pragma unroll
      for (int i = 0; i < CS / 2; i += 2)
        st_shared_b32(z_u32 + act_off(row_of(i), (int)rank * CS + col_of(i)),
                      ptx::cvt_bf16x2(fmaxf(d[i] + bp1[col_of(i)], 0.f), fmaxf(d[i + 1] + bp1[col_of(i + 1)], 0.f)));
      rg.release(rg.prev, lane);
      rg.prev = -1;
    }
    cons_sync();
    send_slice(z_u32, (int)rank * CS, CS, &zbar);
    expect(&zbar, (kCL - 1) * kM * CS * 2);
    wait_z();
    {
      float d[kQc / 2];
      const uint32_t last = product<kQc>(
          d, rg, KS, [&](int c, uint32_t) -> uint32_t { return z_u32 + c * kTile; }, no_pre, fr, fk, lane);
      const float* bp2 = reinterpret_cast<const float*>(ring + (last - ring_u32) + kQc * 128);
      float v[kQc / 2];
#pragma unroll
      for (int i = 0; i < kQc / 2; i++) v[i] = d[i] + bp2[col_of(i)];
      rg.release(rg.prev, lane);
      rg.prev = -1;
      // logits of row r go to CTA r / 8: [8 rows][256] fp32 in its aux buffer
      const uint32_t lb = ptx::smem_u32(&lbar);
#pragma unroll
      for (int i = 0; i < kQc / 2; i += 2) {
        const int row = row_of(i), col = col_of(i);
        const uint32_t dst = (uint32_t)rank;
        const uint32_t off = a_u32 + (uint32_t)(((row & 7) * kQ + (int)rank * kQc + col) * 4);
        const uint32_t g = (uint32_t)(row >> 3);
        if (g == dst) {
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(off), "f"(v[i]), "f"(v[i + 1]) : "memory");
        } else {
          const uint32_t delta = pdelta[(g - rank - 1) & (kCL - 1)];
          st_async_v2(off + delta, __float_as_uint(v[i]), __float_as_uint(v[i + 1]), lb + delta);
        }
        if (p.logits_out && row < nu && istep < s_n[row]) {
          float* o = p.logits_out + ((size_t)(u0 + row) * p.max_n + istep) * kQ + rank * kQc + col;
          o[0] = v[i];
          o[1] = v[i + 1];
        }
      }
    }
    cons_sync();
    expect(&lbar, (kCL - 1) * 8 * kQc * 4);
    ptx::mbar_wait(&lbar, lph);
    lph ^= 1u;
    // ---------------- pick: warp w takes rows 8 rank + 2w, + 1 ----------------
#pragma unroll 1
    for (int jr = 0; jr < 2; jr++) {
      const int j = 2 * warp + jr, row = 8 * (int)rank + j;
      const float* lrow = reinterpret_cast<const float*>(abuf) + j * kQ;
      const int q0 = lane * 8;
      float lg8[8];
      {
        const float4 l0 = *reinterpret_cast<const float4*>(lrow + q0);
        const float4 l1 = *reinterpret_cast<const float4*>(lrow + q0 + 4);
        lg8[0] = l0.x; lg8[1] = l0.y; lg8[2] = l0.z; lg8[3] = l0.w;
        lg8[4] = l1.x; lg8[5] = l1.y; lg8[6] = l1.z; lg8[7] = l1.w;
      }
      float best = -INFINITY;
      int bi = 0x7fffffff;
#pragma unroll
      for (int k = 0; k < 8; k++)
        if (lg8[k] > best) { best = lg8[k]; bi = q0 + k; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      int pick = bi;
      if (p.mode == WNB_MODE_SAMPLING) {
        float uni;
        if (p.uniforms) {
          uni = p.uniforms[(size_t)min(u0 + row, p.B - 1) * p.max_n + min(istep, p.i_last)];
        } else {
          uint32_t rr[4];
          philox4x32_10((uint32_t)istep, (uint32_t)(u0 + row), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), rr);
          uni = (float)(rr[0] >> 8) * (1.0f / 16777216.0f);
        }
        float ex[8];
        float lsum = 0.f;
        int lnz = -1;
#pragma unroll
        for (int k = 0; k < 8; k++) {
          ex[k] = expf(lg8[k] - best);
          lsum += ex[k];
          if (ex[k] > 0.f) lnz = q0 + k;
        }
        float incl = lsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        pick = sample_pick(incl, lsum, lnz, uni, lane, [&](float start, float target) {   // (common.cuh)
          int c = -1;
#pragma unroll
          for (int k = 7; k >= 0; k--) {
            float ck = start;
#pragma unroll
            for (int m = 0; m <= k; m++) ck += ex[m];
            if (ck > target && ex[k] > 0.f) c = q0 + k;
          }
          return c;
        });
      }
      if (lane == 0) {
        if (row < nu && istep < s_n[row]) p.xs[(size_t)(u0 + row) * stride_xs + pos + 1] = pick;
        const uint32_t hp = ptx::smem_u32(&hist[(pos + 1) & 3][row]);
        st_shared_b32(hp, (uint32_t)pick);
        const uint32_t pb = ptx::smem_u32(&pbar);
#pragma unroll
        for (int i = 0; i < kCL - 1; i++) st_async_b32(hp + pdelta[i], (uint32_t)pick, pb + pdelta[i]);
      }
    }
    cons_sync();
    expect(&pbar, (kCL - 1) * 8 * 4);
    ptx::mbar_wait(&pbar, pph);
    pph ^= 1u;
  }
  ptx::cluster_sync();
}

}  // namespace db

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static bool db_shape_ok(int R, int S) { return (R == 256 && S == 256) || (R == 512 && (S == 256 || S == 512)); }
static int db_stage_bytes(int R, int S) {
  const int NG = R / 4, NR = R / 8 + S / 8;
  int b = NG * 128 + db::kTile;                     // W1 chunk + tap tile (the largest chunk)
  b = b > NR * 128 + NR * 4 ? b : NR * 128 + NR * 4;
  return (b + 1023) / 1024 * 1024;
}
static size_t db_fixed_smem(int R, int Ap) { return 1024 + (size_t)2 * R * 128 + (size_t)db_aux_k(Ap) * 128; }
// ring stages that fit next to the activation buffers (0 when fewer than 3)
static int db_stages(int R, int S, int Ap) {
  const long avail = (long)db::kSmemLimit - db::kStaticSmem - (long)db_fixed_smem(R, Ap);
  int n = (int)(avail / db_stage_bytes(R, S));
  if (n > db::kMaxStages) n = db::kMaxStages;
  return n >= 3 ? n : 0;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

WNB_API int wnb_decode_bf16_supported(int Q, int Ap, int R, int S, int ks, int L) {
  if (Q != db::kQ || (ks != 2 && ks != 3) || Ap < 1 || Ap > 256 || Ap % 32 != 0 || L < 1 || L > db::kMaxL) return 0;
  if (!db_shape_ok(R, S)) return 0;
  return db_stages(R, S, Ap) >= 3 ? 1 : 0;
}

// bf16 elements of the packed stream: 8 per-CTA streams back to back.  CTA r's stream, with CR = R/8, CS = S/8,
// Ak = Ap rounded up to 64, every matrix chunk a [N rows][64 k] bf16 tile in the 128B swizzle (element (n, k) at
// n * 64 + ((k / 8) ^ (n % 8)) * 8 + k % 8), K-major:
//   per layer l:  gate chunks  W1 rows [sigmoid of channels r CR .. | tanh of the same], K = [aux Ak | taps j = 0 ..
//                 ks-2 | x(t)] (zero columns past Ap), then b1 of those rows (2 CR fp32);
//                 res chunks   W2 rows [res of channels r CR .. | skip of channels r CS ..], K = R, then their b2 (fp32)
//   post:         post-1 rows r CS .. (K = S) + bp1 slice (fp32), post-2 rows 32 r .. (K = S) + bp2 slice (fp32)
// (the fp32 biases travel as pairs of 16-bit elements).  nets/wavenet.py::_decode_bf16_pack builds it.
WNB_API size_t wnb_decode_bf16_weights(int Q, int Ap, int R, int S, int ks, int L) {
  (void)Q;
  if (R % 64 || S % 64 || Ap < 1 || ks < 1 || L < 1) return 0;
  return ((size_t)L * db_cta_bytes(Ap, R, S, ks) + db_post_bytes(S)) * db::kCL / 2;
}

// bytes of the dilation queues of B utterances: ceil(B / 64) clusters x sum_l (ks-1) d_l slots x R x 64 bf16
WNB_API size_t wnb_decode_bf16_workspace(int B, int R, int ks, const int32_t* host_dilations, int L) {
  if (B < 1 || L < 1 || !host_dilations) return 0;
  size_t slots = 0;
  for (int l = 0; l < L; l++) slots += (size_t)(ks - 1) * host_dilations[l];
  return (size_t)cdiv(B, db::kM) * slots * (size_t)R * db::kM * 2;
}

WNB_API int wnb_decode_bf16_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                               const float* bf, const void* weights, const int32_t* host_dilations, int L, void* queues,
                               const int32_t* n_samples, const float* uniforms, float* logits_out, int B, int P,
                               int max_n, int n_pad, int Th, int Q, int A, int Ap, int R, int S, int ks, int U, int mode,
                               uint64_t seed, int pos0, int xs_base, int h_frame0, void* stream_handle) {
  WNB_REQUIRE(B > 0 && P >= 1 && max_n >= 1 && Th >= 1 && Q > 0 && A > 0 && Ap >= A && R > 0 && S > 0 && ks >= 1 &&
                  U >= 0 && L >= 1, "decode_bf16: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && weights && n_samples && queues && host_dilations, "decode_bf16: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_bf16: U>0 needs upsampling weight and bias");
  WNB_REQUIRE(mode == WNB_MODE_ARGMAX || mode == WNB_MODE_SAMPLING, "decode_bf16: mode should be sampling or argmax");
  if (!wnb_decode_bf16_supported(Q, Ap, R, S, ks, L)) {
    set_error("decode_bf16: shape not covered (Q %d, Ap %d, R %d, S %d, ks %d, L %d): needs Q 256, ks 2 or 3, Ap <= 256, "
              "R/S 256/256, 512/256 or 512/512, L <= %d", Q, Ap, R, S, ks, L, db::kMaxL);
    return WNB_ERR_UNSUPPORTED;
  }
  db::Params p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf;
  p.weights = (const unsigned char*)weights; p.queues = (unsigned char*)queues;
  p.n_samples = n_samples; p.uniforms = uniforms; p.logits_out = logits_out;
  p.B = B; p.P = P; p.max_n = max_n; p.n_pad = n_pad; p.Th = Th; p.A = A; p.Ak = db_aux_k(Ap); p.U = U; p.mode = mode;
  p.L = L; p.ks = ks; p.seed = seed;
  DecodeWindow win;
  if (!decode_window("decode_bf16", P, n_pad, U, ks, max_n, Th, pos0, xs_base, h_frame0, &win)) return WNB_ERR_INVALID;
  p.pos0 = win.pos0; p.i0 = win.i0; p.i_last = win.i_last; p.h_last = win.h_last; p.stride_xs = win.stride_xs;
  p.xs = shift_ptr(xs, -(long long)xs_base); p.h = shift_ptr(h, -(long long)h_frame0);
  p.uniforms = shift_ptr(uniforms, -(long long)win.i0); p.logits_out = shift_ptr(logits_out, -(long long)win.i0 * Q);
  p.nstage = db_stages(R, S, Ap);
  p.stage_bytes = db_stage_bytes(R, S);
  int ncl;
  db_split(B, &ncl, &p.bc);
  p.cta_bytes = (long long)((size_t)L * db_cta_bytes(Ap, R, S, ks) + db_post_bytes(S));
  long long slots = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1, "decode_bf16: dilations must be positive");
    p.dil[l] = host_dilations[l];
    p.qslot[l] = slots;
    slots += (long long)(ks - 1) * host_dilations[l];
  }
  p.q_cluster = slots * (long long)R * db::kM * 2;
  cudaStream_t st = (cudaStream_t)stream_handle;
  // taps before the start of the sequence read zeros: the queues start cleared (by the first call of a session only;
  // later calls continue from what the previous one left)
  if (pos0 == 0) WNB_CUDA(cudaMemsetAsync(queues, 0, (size_t)ncl * p.q_cluster, st));
  const size_t smem = db_fixed_smem(R, Ap) + (size_t)p.nstage * p.stage_bytes;
  auto launch = [&](auto kernel) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(ncl * db::kCL));
    cfg.blockDim = dim3((unsigned)db::kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = db::kCL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, p);
  };
  cudaError_t le;
  if (R == 256) le = launch(db::decode_bf16_kernel<256, 256>);
  else if (S == 256) le = launch(db::decode_bf16_kernel<512, 256>);
  else le = launch(db::decode_bf16_kernel<512, 512>);
  if (le != cudaSuccess) {
    set_error("decode_bf16: launch failed: %s", cudaGetErrorString(le));
    return WNB_ERR_CUDA;
  }
  WNB_CHECK_LAUNCH("decode_bf16");
  return WNB_OK;
}

}  // extern "C"
