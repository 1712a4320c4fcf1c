// decode_warp.cu -- persistent fast-generate kernel, v3, specialised for the BASELINE arctic shape
// (n_resch 64, n_skipch 512, n_quantize 256, aux <= 32, kernel_size 2; any depth/repeat).
//
// v2 (decode_stream.cu) removed the L2 latency from the chain but still spent ~14k cycles per layer in
// six under-populated phases separated by block-wide barriers.  v3 keeps the weight-stream ring (producer
// warp + cp.async.bulk + mbarriers) and restructures the consumers around WARPS:
//   * the stream is packed in "warp tile" order so that every shared-memory read is a conflict-free,
//     fully used 128-byte wavefront;
//   * gate GEMV (128 x 160): warp w owns gate channels 8w..8w+7 (sigmoid and tanh rows), its lanes split
//     K, and a shuffle reduce-scatter leaves each pre-activation in one lane -> the gate is evaluated in
//     registers, no shared-memory partial sums, no extra barrier;
//   * res GEMV (64 x 64): same scheme; the warp that owns residual channels 8w..8w+7 updates them in place
//     and pushes them into the NEXT layer's dilation queue;
//   * skip GEMV (512 x 64) and the post network: lanes split the OUTPUTS (2 per lane), so the running skip
//     sum of all layers lives in registers for the whole step (python order `0 + s0 + s1 ...` kept);
//   * two barriers per layer instead of six.
// Per step the floor is the shared-memory read of the 8.6 MB of weights (67k cycles) or the L2->smem
// stream, whichever is slower; utterances sharing a CTA (NU = 2, 4) reuse both.
// Numerics identical in kind to v1/v2: fp32 FFMA, precise expf/tanhf, first-max argmax, Philox sampling.
//
// CL = 2 (batches of at most half the SM count): ONE UTTERANCE PER 2-CTA CLUSTER.  The 16 "virtual" consumer warps of the
// single-CTA form are split over the two CTAs (8 each); each CTA streams only ITS warps' half of every matrix
// (4.3 MB instead of 8.6 MB per step through its L2 -> shared-memory path, the measured bound), computes its half of
// every output vector and stores it into BOTH CTAs' shared memory (st.shared::cluster, 64..512 floats per phase);
// the consumer barriers that separate the phases become cluster-wide mbarrier phases (every virtual warp arrives on
// both CTAs' barrier with release.cluster, waits on its own with acquire.cluster).  Same per-warp arithmetic in the
// same order as CL = 1, hence the same logits bit for bit.
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace wnb {
namespace dw {

constexpr int kR = 64, kS = 512, kQ = 256, kAp = 32, kK1 = 160;
// W = consumer warps (8 or 16).  More warps = more latency hiding for the dependent smem->FMA chains
// (the kernel is issue-latency bound, the weight stream is always ahead).
constexpr int kSlot = 32 * 1024;          // ring slot: 32 KB, or 2 * kSlot when the BIG (64 KB) schedule is used
constexpr int kMaxL = 64;
// stream layout per layer (floats), G = 32 / W groups of 4 gate values, H = 16 / W groups of 4 res values:
//   W1 [5 j][W warp][G g][32 lane][4] | W2res [2 j][W warp][H g][32 lane][4] | W2skip [64 k][512]
// (value index of a lane = 4 g + e; skip / post matrices are plain K-major, warp w owns columns 512/W * w ...)
// The biases travel INSIDE the stream, right behind the matrix they belong to, so they land in shared memory
// with the weights (a per-layer __ldg of a bias misses L1 every time: ~700 cycles on the critical path).
constexpr int kW1Floats = 5 * 8 * 32 * 16;       // 20480 (80 KB) -> chunks 32K, 32K, 16K + b1
constexpr int kB1Floats = 128;                   // gate bias, appended to the last W1 chunk
constexpr int kWresFloats = 2 * 8 * 32 * 8;      // 4096  (16 KB) -> 1 chunk (+ b2)
constexpr int kB2Floats = kR + kS;               // res + skip bias, appended to the W2res chunk
constexpr int kWskipFloats = 64 * 8 * 64;        // 32768 (128 KB) -> 4 chunks
constexpr int kOffB1 = kW1Floats, kOffWres = kOffB1 + kB1Floats, kOffB2 = kOffWres + kWresFloats,
              kOffWskip = kOffB2 + kB2Floats;
constexpr int kLayerFloats = kOffWskip + kWskipFloats;
constexpr int kPBiasFloats = kS + kQ;            // post biases: one small chunk ahead of the post matrices
constexpr int kP1Floats = 512 * 8 * 64;          // post1 [512][512]  (1 MB)  -> 32 chunks
constexpr int kP2Floats = 512 * 8 * 32;          // post2 [512][256]  (512 KB)-> 16 chunks

struct Params {
  int32_t* xs; const float* h; const float* up_w; const float* up_b;
  const float *wf, *bf, *b1, *b2, *bp1, *bp2;
  const float* stream;
  float* queues; const int32_t* n_samples; const float* uniforms; float* logits_out;
  int B, P, max_n, n_pad, Th, A, U, mode, L, nslot, split, big;
  int pos0, i0, i_last, h_last, stride_xs;   // the call's window (common.cuh DecodeWindow)
  long long rank_stride;   // cluster form: floats between the two CTAs' streams
  unsigned long long seed;
  int dil[kMaxL];
  long long qoff[kMaxL];
  long long q_per_utt;
  long long* timing;   // optional (debug): 16 cycle counters per CTA, filled by warp 0 lane 0
};

#define WNB_T(slot)                                           \
  do {                                                        \
    if (p.timing && tid == 0) {                               \
      const long long now__ = clock64();                      \
      tacc[slot] += now__ - tlast;                            \
      tlast = now__;                                          \
    }                                                         \
  } while (0)

__device__ __forceinline__ void bulk_g2s(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(ptx::smem_u32(smem)), "l"(gmem), "r"(bytes), "r"(ptx::smem_u32(bar))
               : "memory");
}
template <int W>
__device__ __forceinline__ void cons_sync_w() { asm volatile("bar.sync 1, %0;" ::"n"(W * 32) : "memory"); }

// ---- 2-CTA cluster helpers (CL == 2) ----
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
// Phase hand-over between the two CTAs of a cluster WITHOUT fences: every value a CTA owes its peer is sent with
// st.async (shared::cluster), which completes transaction bytes on an mbarrier in the PEER's shared memory, the way TMA
// does.  A phase of a CTA's mbarrier completes when (a) its own consumer warps have met at a CTA barrier and one thread
// has arrived with the number of bytes the peer owes for this phase (arrive.expect_tx) and (b) those bytes have landed.
// Two mbarriers are used alternately; a CTA can never be more than one phase ahead of its peer, because each phase needs
// the peer's data of that phase.
struct XSync {
  uint32_t bar_local;     // shared::cta address of xbars[0]
  uint32_t bar_remote;    // shared::cluster address of the peer's xbars[0]
  uint32_t n;
  __device__ __forceinline__ uint32_t peer_bar() const { return bar_remote + (n & 1u) * 8u; }
  // arrive(): this CTA's share of the phase is complete and sent; wait(): the peer's share has landed.  Work that does
  // not depend on the peer's data may sit between the two (it hides the ~250-cycle DSMEM latency).
  template <int NTHREADS>
  __device__ __forceinline__ void arrive(int tid, uint32_t expect_bytes) {
    asm volatile("bar.sync 1, %0;" ::"n"(NTHREADS) : "memory");
    if (tid == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_local + (n & 1u) * 8u),
                   "r"(expect_bytes) : "memory");
  }
  template <int NTHREADS>
  __device__ __forceinline__ void sync(int tid, uint32_t expect_bytes) {
    arrive<NTHREADS>(tid, expect_bytes);
    wait();
  }
  __device__ __forceinline__ void wait() {
    const uint32_t bar = bar_local + (n & 1u) * 8u, parity = (n >> 1) & 1u;
    ptx::SpinGuard guard;
    for (;;) {
      uint32_t ok;
      asm volatile(
          "{\n\t.reg .pred P;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
          "selp.b32 %0, 1, 0, P;\n\t}\n"
          : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
      if (ok) break;
      if (guard.expired()) { printf("wnb200: decode cluster hand-over timed out after 20 s\n"); __trap(); }
    }
    n++;
  }
};
// store to this CTA's shared memory and (CL == 2) send the value to the same location of the peer CTA, completing 4
// transaction bytes on the peer's mbarrier of the current phase
template <int CL>
__device__ __forceinline__ void st_both(float* p, float v, uint32_t peer_delta, uint32_t peer_bar) {
  *p = v;
  if constexpr (CL == 2)
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                 ::"r"(ptx::smem_u32(p) + peer_delta), "r"(__float_as_uint(v)), "r"(peer_bar) : "memory");
}

struct Ring {
  unsigned char* base; uint64_t* full; uint64_t* empty; int nslot; int split; int slot_bytes;
  int slot; uint32_t phase;   // current chunk's slot and phase parity, advanced incrementally (no runtime division)
  long long waited;           // debug: cycles spent inside acquire()
  uint32_t* ready;            // number of chunks the gatekeeper warp has seen complete (monotonic)
  uint32_t cidx;              // chunks this thread has consumed / published so far
  __device__ __forceinline__ void advance() {
    if (++slot == nslot) { slot = 0; phase ^= 1u; }
  }
  // consumer: wait until the gatekeeper has published chunk `cidx`.  A plain acquire-load poll of a shared
  // counter (~30 cycles when the data is already there) instead of an mbarrier try_wait (~170 cycles): the
  // gatekeeper warp is the only one that touches the TMA `full` barriers.
  __device__ __forceinline__ const float* acquire() {
    const long long t0 = clock64();
    uint32_t seen;
    ptx::SpinGuard guard;
    for (;;) {
      asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(seen) : "r"(ptx::smem_u32(ready)) : "memory");
      if ((int32_t)(seen - cidx) > 0) break;
      if (guard.expired()) { printf("wnb200: decode ring wait timed out after 20 s\n"); __trap(); }
    }
    waited += clock64() - t0;
    return reinterpret_cast<const float*>(base + (size_t)slot * slot_bytes);
  }
  __device__ __forceinline__ void release() {           // consumer: whole warp done with the current chunk
    __syncwarp();
    if ((threadIdx.x & 31) == 0) ptx::mbar_arrive(&empty[slot]);
    advance();
    cidx++;
  }
  // gatekeeper: observe the TMA completion of the current chunk, then publish it to the consumers
  __device__ __forceinline__ void gate() {
    ptx::mbar_wait(&full[slot], phase);
    cidx++;
    asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(ptx::smem_u32(ready)), "r"(cidx) : "memory");
    advance();
  }
  __device__ __forceinline__ void push(const float* src, uint32_t bytes) {  // producer
    ptx::mbar_wait(&empty[slot], phase ^ 1u);
    ptx::mbar_arrive_expect_tx(&full[slot], bytes);
    // several smaller bulk copies per chunk keep more L2 requests in flight than one large copy
    const uint32_t part = bytes / split;
    for (int i = 0; i < split; i++)
      bulk_g2s(base + (size_t)slot * slot_bytes + (size_t)i * part, reinterpret_cast<const unsigned char*>(src) + (size_t)i * part,
               part, &full[slot]);
    advance();
  }
};

// Recursive-halving reduce-scatter over the 32 lanes of a warp: every lane contributes v[0..NV); afterwards
// the total of value j is written to dst[j] by exactly one lane.  NV in {8, 16, 32, 64}.
template <int NV>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[NV], float* dst, int lane) {
  int base = 0;
  if constexpr (NV >= 2) {
#pragma unroll
    for (int lvl = 0; lvl < 5; lvl++) {
      const int off = 16 >> lvl;
      const int n = NV >> lvl;        // values held before this level
      if (n >= 2) {
        const int half = n >> 1;
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int t = 0; t < NV / 2; t++) {
          if (t < half) {
            const float send = up ? v[t] : v[t + half];
            const float keep = up ? v[t + half] : v[t];
            v[t] = keep + __shfl_xor_sync(0xffffffffu, send, off);
          }
        }
        base += up ? half : 0;
      } else {
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
      }
    }
  }
  constexpr int kLeft = (NV >= 32) ? NV / 32 : 1;           // values per lane at the end
  constexpr int kDup = (NV >= 32) ? 1 : 32 / NV;            // lanes holding the same total
  if ((lane & (kDup - 1)) == 0) {
#pragma unroll
    for (int t = 0; t < kLeft; t++) dst[base + t] = v[t];
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

template <int NU, int W, bool BIG, int CL>
__global__ void __launch_bounds__((W / CL) * 32 + 64, 1) decode_warp_kernel(const Params p) {
  static_assert(CL == 1 || (CL == 2 && NU == 1 && W == 16), "cluster form: one utterance per CTA pair, 16 virtual warps");
  constexpr int WP = W / CL;             // physical consumer warps of this CTA (W = virtual warps of the utterance group)
  constexpr int kCons = WP * 32;         // consumer threads
  constexpr int kSlotB = BIG ? 2 * kSlot : kSlot;   // bytes per ring slot
  constexpr int KPC = (BIG ? 32 : 16) * CL;   // skip / post-1 rows (k) per chunk; post-2 has 2 * KPC
  constexpr int kSrow = kS / CL, kQrow = kQ / CL;   // columns of a skip / post-1 / post-2 row in THIS CTA's stream
  constexpr int kLayerF = kLayerFloats - (CL - 1) * (kW1Floats / 2 + kWresFloats / 2 + kWskipFloats / 2);
  constexpr int kJBlock = WP * 2 * (kR / W) * 32;   // floats of one W1 j-block in this CTA's stream
  constexpr bool kW1One = BIG && CL == 2;           // the halved W1 (40.5 KB with b1) fits one 64 KB slot: one acquire
  constexpr int CH = kR / W;             // gate / residual channels owned by a warp (8 or 4)
  constexpr int GV = 2 * CH;             // gate values per lane: [sigmoid CH | tanh CH]
  constexpr int SV = kS / W;             // skip / post-1 outputs per warp (64 or 32)
  constexpr int SL = SV / 32;            // ... per lane (2 or 1)
  constexpr int QV = kQ / W;             // logits per warp (32 or 16)
  constexpr int KS = 32 / QV;            // post-2: lanes sharing one logit split K this many ways (1 or 2)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int L = p.L;
  unsigned char* ring_base = smem_raw;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring_base + (size_t)p.nslot * kSlotB);
  uint64_t* empty = full + p.nslot;
  uint32_t* ready = reinterpret_cast<uint32_t*>(empty + p.nslot);   // + 3 pad words (keeps 16 B alignment)
  float* fw = reinterpret_cast<float*>(ready + 4);
  float* cur = fw;                          // [NU][64]
  float* zs0 = cur + NU * kR;               // [2][NU][64]: gate outputs of even / odd blocks (the peer CTA of a cluster
  float* hcol = zs0 + 2 * NU * kR;          //               may already send block l+1's while block l's are being read)
  float* skipx = hcol + NU * kAp;           // [NU][512]  relu(skip sum) / post hidden input
  float* h1 = skipx + NU * kS;              // [NU][512]
  float* logit = h1 + NU * kS;              // [NU][256]
  float* pre_s = logit + NU * kQ;           // [W warps][GV*NU]   (= 128*NU floats for any W)
  float* qtap = pre_s + 128 * NU;           // [NU][L][64]
  __shared__ int s_n[NU];
  __shared__ __align__(8) uint64_t xbars[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (CL == 2) ? (int)cluster_ctarank() : 0;
  const int vw = rank * WP + warp;          // virtual warp: owns gate channels CH*vw.., skip columns SV*vw.., logits QV*vw..
  const int u0 = (blockIdx.x / CL) * NU;
  const int stride_xs = p.stride_xs;

  if (tid == 0) {
    for (int i = 0; i < p.nslot; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], WP);
    }
    if (CL == 2) { ptx::mbar_init(&xbars[0], 1); ptx::mbar_init(&xbars[1], 1); }
    *ready = 0u;
    ptx::fence_barrier_init();
  }
  if (tid < NU) s_n[tid] = (u0 + tid < p.B) ? p.i0 + p.n_samples[u0 + tid] : 0;   // absolute end
  __syncthreads();
  int nmax = 0;
#pragma unroll
  for (int u = 0; u < NU; u++) nmax = max(nmax, s_n[u]);
  if (nmax <= p.i0) return;
  XSync xs_{0u, 0u, 0u};
  uint32_t peer_delta = 0;
  if constexpr (CL == 2) {
    // both CTAs must have initialised their barriers before the first remote arrival: hardware cluster barrier, once
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    xs_.bar_local = ptx::smem_u32(&xbars[0]);
    xs_.bar_remote = mapa_u32(xs_.bar_local, (uint32_t)(rank ^ 1));
    peer_delta = xs_.bar_remote - xs_.bar_local;
  }
  // barrier between phases: the consumer warps of this CTA (CL == 1) or the hand-over of `floats` values per CTA
  // between the two CTAs of the cluster (CL == 2)
  auto phase_sync = [&](int floats) {
    if constexpr (CL == 2) xs_.template sync<kCons>(tid, (uint32_t)floats * 4u); else cons_sync_w<W>();
  };
  auto phase_arrive = [&](int floats) {   // split form: (CL == 1: nothing to send, the barrier happens in phase_wait)
    if constexpr (CL == 2) xs_.template arrive<kCons>(tid, (uint32_t)floats * 4u);
  };
  auto phase_wait = [&]() {
    if constexpr (CL == 2) xs_.wait(); else cons_sync_w<W>();
  };
  const float* my_stream = p.stream + (size_t)rank * p.rank_stride;
  const int last_pos = p.P - 1 + nmax - 1;
  Ring ring{ring_base, full, empty, p.nslot, p.split, kSlotB, 0, 0u, 0ll, ready, 0u};

  if (warp == WP) {
    // ================================ producer warp ================================
    if (lane == 0) {
      for (int pos = p.pos0; pos <= last_pos; pos++) {
        const bool want = pos >= p.P - 1;
        for (int l = 0; l < L; l++) {
          const float* base = my_stream + (size_t)l * kLayerF;
          if (kW1One) {
            // W1 j = 0..4 | b1 | W2res | b2: ONE 51.8 KB chunk per block (they are contiguous in the stream), so that the
            // three 64 KB slots hold [this block's gate+res][this block's skip][NEXT block's gate+res]: the stream runs
            // half a block further ahead than with a slot each for W1 and W2res
            ring.push(base, (5 * kJBlock + kB1Floats + kWresFloats / CL + kB2Floats) * 4);
          } else {
            if (BIG) {
              ring.push(base, 4 * kJBlock * 4);                            // W1 j = 0..3
            } else {
              ring.push(base, 2 * kJBlock * 4);                            // W1 j = 0,1
              ring.push(base + 2 * kJBlock, 2 * kJBlock * 4);              // W1 j = 2,3
            }
            ring.push(base + 4 * kJBlock, (kJBlock + kB1Floats) * 4);      // W1 j = 4, then b1
          }
          const float* wres = base + 5 * kJBlock + kB1Floats;
          if (!kW1One) ring.push(wres, (kWresFloats / CL + kB2Floats) * 4);   // W2res, then b2
          if (want)
            for (int c = 0; c < 64 / KPC; c++)
              ring.push(wres + kWresFloats / CL + kB2Floats + c * (KPC * kSrow), KPC * kSrow * 4);
        }
        if (want) {
          const float* pb = my_stream + (size_t)L * kLayerF;
          ring.push(pb, kPBiasFloats * 4);                                 // bp1 | bp2
          const float* p1 = pb + kPBiasFloats;
          for (int c = 0; c < kS / KPC; c++) ring.push(p1 + (size_t)c * (KPC * kSrow), KPC * kSrow * 4);
          const float* p2 = p1 + kP1Floats / CL;
          for (int c = 0; c < kS / (2 * KPC); c++) ring.push(p2 + (size_t)c * (2 * KPC * kQrow), 2 * KPC * kQrow * 4);
        }
      }
    }
    return;
  }
  if (warp == WP + 1) {
    // ================================ gatekeeper warp ================================
    if (lane == 0) {
      const int per_layer_warm = kW1One ? 1 : ((BIG ? 2 : 3) + 1), per_layer_skip = 64 / KPC;
      const int post_chunks = 1 + kS / KPC + kS / (2 * KPC);
      for (int pos = p.pos0; pos <= last_pos; pos++) {
        const bool want = pos >= p.P - 1;
        const int n = L * (per_layer_warm + (want ? per_layer_skip : 0)) + (want ? post_chunks : 0);
        for (int i = 0; i < n; i++) ring.gate();
      }
    }
    return;
  }

  // ================================ consumer warps ================================
  // aux column and every block's dilation-queue tap for time step `pos_t`, by threads t0, t0 + nt, ...  (used by the step
  // prologue, and -- for the NEXT step -- by the warps that are idle while warp 0 picks the sample: neither depends on it)
  auto fetch_aux_taps = [&](int pos_t, int t0, int nt) {
    for (int e = t0; e < NU * kAp; e += nt) {
      const int u = e >> 5, a = e & 31;
      const int ug = min(u0 + u, p.B - 1);
      float v = 0.f;
      if (a < p.A) {
        const int j = max(pos_t - p.n_pad, 0);
        if (p.U > 0) {
          const int tf = min(j / p.U, p.h_last), jj = j % p.U;
          v = fmaf(__ldg(p.h + ((size_t)ug * p.A + a) * p.Th + tf), __ldg(p.up_w + jj), __ldg(p.up_b));
        } else {
          v = __ldg(p.h + ((size_t)ug * p.A + a) * p.Th + min(j, p.h_last));
        }
      }
      hcol[e] = v;
    }
    for (int e = t0; e < NU * L * kR; e += nt) {
      const int r = e & 63;
      const int ul = e >> 6;                                 // u * L + l  (no runtime division: NU <= 4)
      const int u = (ul >= L) + (ul >= 2 * L) + (ul >= 3 * L);
      const int l = ul - u * L;
      const int ug = min(u0 + u, p.B - 1);
      const int d = p.dil[l];
      float v = 0.f;
      // tap = this layer's input at time pos_t - d: ring slot (pos_t - d) % d == pos_t % d, i.e. the slot that is
      // overwritten with the time-`pos_t` input later in THAT step -> all reads happen before its first barrier
      if (pos_t - d >= 0) {
        const float* q = p.queues + (size_t)ug * p.q_per_utt + p.qoff[l];
        v = __ldcg(q + (size_t)(pos_t & (d - 1)) * kR + r);
      }
      qtap[e] = v;
    }
  };
  bool have_next = false;    // hcol / qtap already hold the next step's values (prefetched during the pick)
  float uni_next = 0.f;      // sampling: the uniform of generated sample `uni_for`, drawn one step ahead
  int uni_for = -1;
  float* my_pre = pre_s + warp * GV * NU;
  long long tacc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  long long tlast = clock64();
  for (int pos = p.pos0; pos <= last_pos; pos++) {
    const bool want = pos >= p.P - 1;
    if (pos == p.P - 1 && p.timing && tid == 0) {   // time only the free-running steps
      for (int i = 0; i < 12; i++) tacc[i] = 0;
      tlast = clock64();
      ring.waited = 0;
    }
    // ---- step prologue: front gather, aux column, all queue taps ----
    for (int e = tid; e < NU * kR; e += kCons) {
      const int u = e >> 6, r = e & 63;
      const int ug = min(u0 + u, p.B - 1);
      float v = __ldg(p.bf + r);
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int pp = pos - (1 - k);
        if (pp >= 0) {
          int q = p.xs[(size_t)ug * stride_xs + pp] % kQ;
          if (q < 0) q += kQ;
          v += __ldg(p.wf + ((size_t)k * kQ + q) * kR + r);
        }
      }
      cur[e] = v;
    }
    if (!have_next) fetch_aux_taps(pos, tid, kCons);
    have_next = false;
    WNB_T(0);
    cons_sync_w<WP>();     // (CTA-local: the prologue only touches this CTA's shared memory)
    WNB_T(1);

    float skip_tot[NU][SL];
#pragma unroll
    for (int u = 0; u < NU; u++)
#pragma unroll
      for (int e = 0; e < SL; e++) skip_tot[u][e] = 0.f;

    for (int l = 0; l < L; l++) {
      float* zs = zs0 + (l & 1) * NU * kR;
      // ---------------- phase A: gate pre-activations, split K over lanes ----------------
      float acc[NU * GV];
#pragma unroll
      for (int i = 0; i < NU * GV; i++) acc[i] = 0.f;
      const float* chunk = nullptr;
      float gate_bs = 0.f, gate_bt = 0.f;
#pragma unroll
      for (int j = 0; j < 5; j++) {
        if (j == 0 || (!kW1One && ((!BIG && j == 2) || j == 4))) chunk = ring.acquire();
        // [j][warp][group g][lane][4]: consecutive lanes read consecutive 16 B -> conflict-free LDS.128
        const int jj = kW1One ? j : ((j == 4) ? 0 : (BIG ? j : (j & 1)));   // index of this j inside its chunk
        const float4* wp = reinterpret_cast<const float4*>(chunk + (size_t)(jj * WP + warp) * (GV * 32)) + lane;
        float4 wv[GV / 4];
#pragma unroll
        for (int g = 0; g < GV / 4; g++) wv[g] = wp[g * 32];
#pragma unroll
        for (int u = 0; u < NU; u++) {
          const float x = (j < 2) ? qtap[((size_t)u * L + l) * kR + (j * 32 + lane)]
                                  : (j < 4) ? cur[u * kR + (j - 2) * 32 + lane] : hcol[u * kAp + lane];
          float* a = acc + u * GV;
#pragma unroll
          for (int g = 0; g < GV / 4; g++) {
            a[4 * g] = fmaf(wv[g].x, x, a[4 * g]); a[4 * g + 1] = fmaf(wv[g].y, x, a[4 * g + 1]);
            a[4 * g + 2] = fmaf(wv[g].z, x, a[4 * g + 2]); a[4 * g + 3] = fmaf(wv[g].w, x, a[4 * g + 3]);
          }
        }
        if (j == 4) {   // b1 sits right behind the j = 4 weights in this chunk
          const int c = vw * CH + (lane % CH);
          gate_bs = chunk[(kW1One ? 5 : 1) * kJBlock + c];
          gate_bt = chunk[(kW1One ? 5 : 1) * kJBlock + 64 + c];
        }
        if (!kW1One && ((!BIG && j == 1) || j == 3 || j == 4)) ring.release();   // (kW1One: released after phase B)
      }
      WNB_T(2);
      warp_reduce_scatter<NU * GV>(acc, my_pre, lane);
      __syncwarp();
      if (lane < CH * NU) {   // (splitting sigmoid / tanh over two lane groups was measured: divergence serialises them)
        const int u = lane / CH, cc = lane % CH, c = vw * CH + cc;
        const float a = my_pre[u * GV + cc] + gate_bs;
        const float g = my_pre[u * GV + CH + cc] + gate_bt;
        st_both<CL>(&zs[u * kR + c], sigmoidf_(a) * tanhf(g), peer_delta, xs_.peer_bar());
      }
      WNB_T(3);
      // CL == 2: the K half of the residual GEMV that multiplies THIS CTA's gate channels runs while the peer's half of z
      // is in flight; the other half follows the wait
      phase_arrive(NU * kR / 2);
      if constexpr (CL == 1) phase_wait();
      WNB_T(4);
      // ---------------- phase B: residual 1x1 (split K) ----------------
      float skip_b[SL];
      {
        float racc[NU * CH];
#pragma unroll
        for (int i = 0; i < NU * CH; i++) racc[i] = 0.f;
        const float* rc = kW1One ? chunk + 5 * kJBlock + kB1Floats : ring.acquire();   // (kW1One: same chunk as W1)
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          const int j = (CL == 2) ? (jj ^ rank) : jj;
          if (CL == 2 && jj == 1) phase_wait();
          const float4* wp = reinterpret_cast<const float4*>(rc + (size_t)(j * WP + warp) * (CH * 32)) + lane;
          float4 wv[CH / 4];
#pragma unroll
          for (int g = 0; g < CH / 4; g++) wv[g] = wp[g * 32];
#pragma unroll
          for (int u = 0; u < NU; u++) {
            const float x = zs[u * kR + j * 32 + lane];
            float* a = racc + u * CH;
#pragma unroll
            for (int g = 0; g < CH / 4; g++) {
              a[4 * g] = fmaf(wv[g].x, x, a[4 * g]); a[4 * g + 1] = fmaf(wv[g].y, x, a[4 * g + 1]);
              a[4 * g + 2] = fmaf(wv[g].z, x, a[4 * g + 2]); a[4 * g + 3] = fmaf(wv[g].w, x, a[4 * g + 3]);
            }
          }
        }
        // b2 = [res 64 | skip 512] sits right behind the res weights in this chunk
        const float res_b = rc[kWresFloats / CL + vw * CH + (lane % CH)];
#pragma unroll
        for (int e = 0; e < SL; e++) skip_b[e] = rc[kWresFloats / CL + kR + vw * SV + lane * SL + e];
        ring.release();
        warp_reduce_scatter<NU * CH>(racc, my_pre, lane);
        __syncwarp();
        if (lane < CH * NU) {
          const int u = lane / CH, cc = lane % CH, c = vw * CH + cc;
          // Layer 0's input (the front output) goes into its queue here, not in the prologue: the slot is the one this step's
          // taps were read from, and with CL == 2 the peer reads them while picking the previous sample (the next-step
          // prefetch) -- a peer already in this step's prologue could overwrite the slot under that read.  Past the z
          // hand-over of layer 0 both CTAs have read all their taps; each writes its own channels, like the other layers.
          if (l == 0 && u0 + u < p.B) {
            float* q0 = p.queues + (size_t)(u0 + u) * p.q_per_utt + p.qoff[0];
            __stcg(q0 + (size_t)(pos & (p.dil[0] - 1)) * kR + c, cur[u * kR + c]);
          }
          const float v = my_pre[u * CH + cc] + res_b + cur[u * kR + c];
          st_both<CL>(&cur[u * kR + c], v, peer_delta, xs_.peer_bar());
          if (l + 1 < L && u0 + u < p.B) {   // input of layer l+1 at time `pos` -> its dilation queue
            float* q = p.queues + (size_t)(u0 + u) * p.q_per_utt + p.qoff[l + 1];
            __stcg(q + (size_t)(pos & (p.dil[l + 1] - 1)) * kR + c, v);   // dilations are powers of two
          }
        }
      }
      WNB_T(5);
      phase_arrive(NU * kR / 2);   // the residual outputs travel to the peer while the skip GEMV runs
      // ---------------- phase B': skip 1x1, lanes own outputs SV*warp + SL*lane (+e) ----------------
      if (want) {
        // (CL == 2 leaves 2 warps per scheduler: a single accumulator per output would make the K loop one dependent
        //  FMA chain nobody hides; even / odd k go to two accumulators that are added at the end)
        float s[NU][SL], s_odd[NU][SL];
#pragma unroll
        for (int u = 0; u < NU; u++)
#pragma unroll
          for (int e = 0; e < SL; e++) { s[u][e] = 0.f; s_odd[u][e] = 0.f; }
#pragma unroll 1
        for (int c4 = 0; c4 < 64 / KPC; c4++) {
          const float* sc = ring.acquire() + warp * SV + lane * SL;   // (column inside this CTA's kSrow-wide rows)
#pragma unroll
          for (int k4 = 0; k4 < KPC; k4 += 4) {
            float4 zv[NU];
#pragma unroll
            for (int u = 0; u < NU; u++) zv[u] = *reinterpret_cast<const float4*>(zs + u * kR + c4 * KPC + k4);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
              float wv[SL];
              if constexpr (SL == 2) {
                const float2 t2 = *reinterpret_cast<const float2*>(sc + (size_t)(k4 + kk) * kSrow);
                wv[0] = t2.x; wv[1] = t2.y;
              } else {
                wv[0] = sc[(size_t)(k4 + kk) * kSrow];
              }
#pragma unroll
              for (int u = 0; u < NU; u++) {
                const float z = kk == 0 ? zv[u].x : kk == 1 ? zv[u].y : kk == 2 ? zv[u].z : zv[u].w;
#pragma unroll
                for (int e = 0; e < SL; e++) {
                  if (CL == 2 && (kk & 1)) s_odd[u][e] = fmaf(wv[e], z, s_odd[u][e]);
                  else s[u][e] = fmaf(wv[e], z, s[u][e]);
                }
              }
            }
          }
          ring.release();
        }
#pragma unroll
        for (int e = 0; e < SL; e++) {
          const float bv = skip_b[e];
#pragma unroll
          for (int u = 0; u < NU; u++) {
            const float sv = (CL == 2 ? s[u][e] + s_odd[u][e] : s[u][e]) + bv;
            skip_tot[u][e] = (l == 0) ? sv : skip_tot[u][e] + sv;   // python `0 + s0 + s1 ...`, wavenet.py:374
          }
        }
      }
      WNB_T(6);
      phase_wait();
      WNB_T(7);
    }

    if (want) {
      // ---------------- post network ----------------
#pragma unroll
      for (int u = 0; u < NU; u++)
#pragma unroll
        for (int e = 0; e < SL; e++)
          st_both<CL>(&skipx[u * kS + vw * SV + lane * SL + e], fmaxf(skip_tot[u][e], 0.f), peer_delta, xs_.peer_bar());
      float post_b1[SL], post_b2;
      {
        const float* pbias = ring.acquire();   // [bp1 512 | bp2 256]
#pragma unroll
        for (int e = 0; e < SL; e++) post_b1[e] = pbias[vw * SV + lane * SL + e];
        post_b2 = pbias[kS + vw * QV + (lane % QV)];
        ring.release();
      }
      phase_sync(NU * kS / 2);
      {
        float s[NU][SL], s_odd[NU][SL];
#pragma unroll
        for (int u = 0; u < NU; u++)
#pragma unroll
          for (int e = 0; e < SL; e++) { s[u][e] = 0.f; s_odd[u][e] = 0.f; }
#pragma unroll 1
        for (int c = 0; c < kS / KPC; c++) {
          const float* pc = ring.acquire() + warp * SV + lane * SL;
#pragma unroll
          for (int k4 = 0; k4 < KPC; k4 += 4) {
            float4 xv[NU];
#pragma unroll
            for (int u = 0; u < NU; u++) xv[u] = *reinterpret_cast<const float4*>(skipx + u * kS + c * KPC + k4);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
              float wv[SL];
              if constexpr (SL == 2) {
                const float2 t2 = *reinterpret_cast<const float2*>(pc + (size_t)(k4 + kk) * kSrow);
                wv[0] = t2.x; wv[1] = t2.y;
              } else {
                wv[0] = pc[(size_t)(k4 + kk) * kSrow];
              }
#pragma unroll
              for (int u = 0; u < NU; u++) {
                const float x = kk == 0 ? xv[u].x : kk == 1 ? xv[u].y : kk == 2 ? xv[u].z : xv[u].w;
#pragma unroll
                for (int e = 0; e < SL; e++) {
                  if (CL == 2 && (kk & 1)) s_odd[u][e] = fmaf(wv[e], x, s_odd[u][e]);
                  else s[u][e] = fmaf(wv[e], x, s[u][e]);
                }
              }
            }
          }
          ring.release();
        }
#pragma unroll
        for (int e = 0; e < SL; e++) {
          const float bv = post_b1[e];
#pragma unroll
          for (int u = 0; u < NU; u++)
            st_both<CL>(&h1[u * kS + vw * SV + lane * SL + e],
                        fmaxf((CL == 2 ? s[u][e] + s_odd[u][e] : s[u][e]) + bv, 0.f), peer_delta, xs_.peer_bar());
        }
      }
      phase_sync(NU * kS / 2);
      WNB_T(8);
      const int i = pos - (p.P - 1);
      {
        // logit o = QV*warp + (lane % QV); when QV == 16 the two half-warps split K (even / odd k)
        const int lo = lane % QV, ksel = lane / QV;
        float s[NU], s_b[NU];
#pragma unroll
        for (int u = 0; u < NU; u++) { s[u] = 0.f; s_b[u] = 0.f; }
#pragma unroll 1
        for (int c = 0; c < kS / (2 * KPC); c++) {
          const float* pc = ring.acquire() + warp * QV + lo;
#pragma unroll
          for (int k4 = 0; k4 < 2 * KPC; k4 += 4) {
            float4 xv[NU];
#pragma unroll
            for (int u = 0; u < NU; u++) xv[u] = *reinterpret_cast<const float4*>(h1 + u * kS + c * (2 * KPC) + k4);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
              if (KS == 1 || (kk & 1) == ksel) {
                const float wv = pc[(size_t)(k4 + kk) * kQrow];
#pragma unroll
                for (int u = 0; u < NU; u++) {
                  const float x = kk == 0 ? xv[u].x : kk == 1 ? xv[u].y : kk == 2 ? xv[u].z : xv[u].w;
                  if (CL == 2 && (kk & 2)) s_b[u] = fmaf(wv, x, s_b[u]);   // (second accumulator: see the skip GEMV)
                  else s[u] = fmaf(wv, x, s[u]);
                }
              }
            }
          }
          ring.release();
        }
        const float bv = post_b2;
#pragma unroll
        for (int u = 0; u < NU; u++) {
          float v = (CL == 2) ? s[u] + s_b[u] : s[u];
          if (KS == 2) v += __shfl_xor_sync(0xffffffffu, v, 16);
          v += bv;
          if (ksel == 0) {
            st_both<CL>(&logit[u * kQ + vw * QV + lo], v, peer_delta, xs_.peer_bar());
            if (p.logits_out && u0 + u < p.B && i < s_n[u])
              p.logits_out[((size_t)(u0 + u) * p.max_n + i) * kQ + vw * QV + lo] = v;
          }
        }
      }
      phase_sync(NU * kQ / 2);
      WNB_T(9);
      // ---------------- pick: warp u handles utterance u; the other warps fetch the next step's aux column and taps ------
      if (warp >= NU && pos < last_pos && kCons > 32 * NU) {
        fetch_aux_taps(pos + 1, tid - 32 * NU, kCons - 32 * NU);
      }
      have_next = pos < last_pos && kCons > 32 * NU;
      if (warp < NU) {
        const int u = warp;
        const int q0 = lane * 8, q1 = q0 + 8;
        float lg8[8];   // this lane's 8 logits: two 16-byte shared-memory loads, kept in registers for all passes
        {
          const float4 l0 = *reinterpret_cast<const float4*>(logit + u * kQ + q0);
          const float4 l1 = *reinterpret_cast<const float4*>(logit + u * kQ + q0 + 4);
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
            uni = p.uniforms[(size_t)min(u0 + u, p.B - 1) * p.max_n + min(i, p.i_last)];
          } else if (uni_for == i) {
            uni = uni_next;            // drawn during the previous step's pick, off the critical path
          } else {
            uint32_t rr[4];
            philox4x32_10((uint32_t)i, (uint32_t)(u0 + u), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), rr);
            uni = (float)(rr[0] >> 8) * (1.0f / 16777216.0f);
          }
          float ex[8];
          float lsum = 0.f;
          int lnz = -1;                         // this lane's last class of nonzero probability
#pragma unroll
          for (int k = 0; k < 8; k++) {
            ex[k] = expf(lg8[k] - best);
            lsum += ex[k];
            if (ex[k] > 0.f) lnz = q0 + k;
          }
          float incl = lsum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          pick = sample_pick(incl, lsum, lnz, uni, lane, [&](float start, float target) {   // (common.cuh)
            int c = -1;
#pragma unroll
            for (int k = 7; k >= 0; k--) {      // first k (ascending) with e > 0 whose running sum passes the target
              float ck = start;
#pragma unroll
              for (int m = 0; m <= k; m++) ck += ex[m];
              if (ck > target && ex[k] > 0.f) c = q0 + k;
            }
            return c;
          });
        }
        // (CL == 2: both CTAs hold the same 256 logits and make the same pick; each writes it -- same value -- so
        //  that its own next prologue reads what it wrote, no cross-CTA dependency on global memory)
        if (lane == 0 && u0 + u < p.B && i < s_n[u]) p.xs[(size_t)(u0 + u) * stride_xs + pos + 1] = pick;
        if (p.mode == WNB_MODE_SAMPLING && !p.uniforms) {   // next step's uniform, while the other warps fetch its taps
          uint32_t rr[4];
          philox4x32_10((uint32_t)(i + 1), (uint32_t)(u0 + u), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), rr);
          uni_next = (float)(rr[0] >> 8) * (1.0f / 16777216.0f);
          uni_for = i + 1;
        }
      }
      cons_sync_w<WP>();
      WNB_T(10);
    }
  }
  if constexpr (CL == 2) {   // no CTA leaves while its peer may still send into its shared memory: a last 1-float hand-over
    if (tid == 0) st_both<CL>(&pre_s[0], 0.f, peer_delta, xs_.peer_bar());
    phase_sync(1);
  }
  if (p.timing && tid == 0) {
    for (int i = 0; i < 12; i++) p.timing[(size_t)blockIdx.x * 16 + i] = tacc[i];
    p.timing[(size_t)blockIdx.x * 16 + 12] = ring.waited;
  }
}

}  // namespace dw

// utterances per CTA, consumer warps and cluster size for a batch of B utterances (shared by the packer and the
// launcher).  Up to half the SM count of utterances: one utterance per 2-CTA cluster, so that 2 B SMs stream the
// weights and every cluster is resident at once (the kernel runs one CTA per SM: more clusters would run as a second
// wave and double the decode time).
static void decode_warp_plan(int B, int* NU, int* W, int* CL) {
  int nu = 1;
  if (B > device_sms() * 2) nu = 4; else if (B > device_sms()) nu = 2;
  *NU = nu;
  *W = (nu == 4) ? 8 : 16;   // 16 warps hide the smem->FMA latency; NU = 4 needs the registers of the 8-warp form
  static const int cl_on = [] { const char* e = getenv("WNB_DECODE_CL"); return (e && e[0] == '1') ? 0 : 1; }();
  *CL = (cl_on && B <= device_sms() / 2) ? 2 : 1;
}

// ring slots for NU utterances per CTA and L layers, given the per-CTA work space: three 64 KB slots (half as many
// mbarrier round trips per step) when they fit and WNB_DECODE_BIG is not 0, else up to six 32 KB slots.  False when
// fewer than three fit.  Shared by the launcher and wnb_decode_warp_form.
static bool decode_warp_slots(int NU, int L, int* nslot, bool* big, size_t* work) {
  using namespace dw;
  *work = ((size_t)NU * (kR * 3 + kAp + 2 * kS + kQ + (size_t)L * kR) + 128 * NU) * sizeof(float);
  const long avail = 227L * 1024 - 256 - (long)*work - 16 * 16;
  const char* eb = getenv("WNB_DECODE_BIG");
  *big = avail >= 3L * 2 * kSlot && !(eb && atoi(eb) == 0);
  int n = *big ? 3 : (int)(avail / kSlot);
  if (n > 6) n = 6;
  *nslot = n;
  return n >= 3;
}

int decode_warp_launch(dw::Params& p, int W_packed, int CL_packed, cudaStream_t st) {
  using namespace dw;
  int NU, W, CL;
  decode_warp_plan(p.B, &NU, &W, &CL);
  if (W != W_packed || CL != CL_packed) {
    set_error("decode_warp: stream packed for %d consumer warps / cluster %d but the plan for B=%d is %d / %d", W_packed,
              CL_packed, p.B, W, CL);
    return WNB_ERR_INVALID;
  }
  p.rank_stride = (long long)((size_t)p.L * (kLayerFloats - (CL - 1) * (kW1Floats / 2 + kWresFloats / 2 + kWskipFloats / 2)) +
                              kPBiasFloats + (kP1Floats + kP2Floats) / CL);
  int nslot;
  bool big;
  size_t work;
  if (!decode_warp_slots(NU, p.L, &nslot, &big, &work)) return WNB_ERR_UNSUPPORTED;
  p.nslot = nslot;
  p.big = big ? 1 : 0;
  {
    const char* e = getenv("WNB_DECODE_SPLIT");
    int sp = e ? atoi(e) : 1;
    if (sp != 1 && sp != 2 && sp != 4 && sp != 8) sp = 1;
    p.split = sp;
  }
  const size_t smem = (size_t)nslot * (big ? 2 * kSlot : kSlot) + 2 * nslot * sizeof(uint64_t) + 16 + work;
  const int grid = cdiv(p.B, NU) * CL;
  auto launch = [&](auto kernel, int threads) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, p);
  };
  cudaError_t le;
  if (CL == 2) le = big ? launch(decode_warp_kernel<1, 16, true, 2>, 8 * 32 + 64) : launch(decode_warp_kernel<1, 16, false, 2>, 8 * 32 + 64);
  else if (NU == 4) le = big ? launch(decode_warp_kernel<4, 8, true, 1>, 8 * 32 + 64) : launch(decode_warp_kernel<4, 8, false, 1>, 8 * 32 + 64);
  else if (NU == 2) le = big ? launch(decode_warp_kernel<2, 16, true, 1>, 16 * 32 + 64) : launch(decode_warp_kernel<2, 16, false, 1>, 16 * 32 + 64);
  else le = big ? launch(decode_warp_kernel<1, 16, true, 1>, 16 * 32 + 64) : launch(decode_warp_kernel<1, 16, false, 1>, 16 * 32 + 64);
  if (le != cudaSuccess) {
    set_error("decode_warp: launch failed: %s", cudaGetErrorString(le));
    return WNB_ERR_CUDA;
  }
  WNB_CHECK_LAUNCH("decode_warp");
  return WNB_OK;
}

}  // namespace wnb

using namespace wnb;

extern "C" {

// floats of the warp-tiled decode stream (layout: csrc/decode_warp.cu header) for L layers and cluster size CL (1 or 2:
// CL per-CTA streams back to back, each with the full biases and 1/CL of every matrix)
WNB_API size_t wnb_decode_warp_floats(int L, int CL) {
  using namespace dw;
  if (CL != 2) CL = 1;
  const size_t per_rank = (size_t)L * (kLayerFloats - (CL - 1) * (kW1Floats / 2 + kWresFloats / 2 + kWskipFloats / 2)) +
                          kPBiasFloats + (kP1Floats + kP2Floats) / CL;
  return per_rank * CL;
}

// debug: device buffer (16 int64 per CTA) that the next wnb_decode_warp_at launches fill with per-phase cycle
// counts of the free-running steps (NULL switches it off).  Slots: 0 prologue, 1 sync, 2 gate GEMV, 3 reduce+gate,
// 4 sync, 5 res GEMV, 6 skip GEMV, 7 sync, 8 post1 (+relu+sync), 9 post2 (+sync), 10 pick (+sync)
static long long* g_decode_timing = nullptr;
WNB_API void wnb_decode_warp_set_timing(long long* buf) { g_decode_timing = buf; }

// 1 when the warp-tiled kernel covers the configuration
WNB_API int wnb_decode_warp_supported(int Q, int Ap, int R, int S, int ks, int L) {
  return (Q == dw::kQ && Ap == dw::kAp && R == dw::kR && S == dw::kS && ks == 2 && L >= 1 && L <= dw::kMaxL) ? 1 : 0;
}

// consumer warps (8 or 16) the launcher will use for B utterances: the stream must be packed accordingly
WNB_API int wnb_decode_warp_plan(int B) {
  int NU, W, CL;
  decode_warp_plan(B, &NU, &W, &CL);
  return W;
}
// CTAs per utterance (cluster size, 1 or 2) the launcher will use for B utterances
WNB_API int wnb_decode_warp_cluster(int B) {
  int NU, W, CL;
  decode_warp_plan(B, &NU, &W, &CL);
  return CL;
}

// the decode_warp_kernel<NU, W, BIG, CL> instantiation the launcher would run for B utterances and L layers, under the
// current WNB_DECODE_BIG: form[0..3] = NU, W, CL, BIG (0 / 1).  WNB_ERR_UNSUPPORTED when no ring fits.
WNB_API int wnb_decode_warp_form(int B, int L, int32_t* form) {
  WNB_REQUIRE(B > 0 && L >= 1 && L <= dw::kMaxL, "decode_warp_form: bad shape");
  WNB_REQUIRE(form, "decode_warp_form: null pointer");
  int NU, W, CL, nslot;
  bool big;
  size_t work;
  decode_warp_plan(B, &NU, &W, &CL);
  if (!decode_warp_slots(NU, L, &nslot, &big, &work)) {
    set_error("decode_warp_form: not enough shared memory for this depth");
    return WNB_ERR_UNSUPPORTED;
  }
  form[0] = NU; form[1] = W; form[2] = CL; form[3] = big ? 1 : 0;
  return WNB_OK;
}

WNB_API int wnb_decode_warp_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                               const float* bf, const float* stream, const float* b1, const float* b2, const float* bp1,
                               const float* bp2, const int32_t* host_dilations, int L, void* queues,
                               const int32_t* n_samples, const float* uniforms, float* logits_out, int B, int P,
                               int max_n, int n_pad, int Th, int A, int U, int mode, uint64_t seed, int W, int CL,
                               int pos0, int xs_base, int h_frame0, void* stream_handle) {
  WNB_REQUIRE(B > 0 && P >= 1 && max_n >= 1 && Th >= 1 && A > 0 && A <= dw::kAp && U >= 0 && L >= 1 && L <= dw::kMaxL,
              "decode_warp: bad shape");
  WNB_REQUIRE(xs && h && wf && bf && stream && b1 && b2 && bp1 && bp2 && n_samples && queues,
              "decode_warp: null pointer");
  WNB_REQUIRE(U == 0 || (up_w && up_b), "decode_warp: U>0 needs upsampling weight and bias");
  WNB_REQUIRE(mode == WNB_MODE_ARGMAX || mode == WNB_MODE_SAMPLING, "decode_warp: mode should be sampling or argmax");
  dw::Params p{};
  p.xs = xs; p.h = h; p.up_w = up_w; p.up_b = up_b; p.wf = wf; p.bf = bf; p.b1 = b1; p.b2 = b2; p.bp1 = bp1;
  p.bp2 = bp2; p.stream = stream; p.queues = (float*)queues; p.n_samples = n_samples; p.uniforms = uniforms;
  p.logits_out = logits_out;
  p.B = B; p.P = P; p.max_n = max_n; p.n_pad = n_pad; p.Th = Th; p.A = A; p.U = U; p.mode = mode; p.L = L;
  p.seed = seed;
  const int Q = dw::kQ;
  DecodeWindow win;
  if (!decode_window("decode_warp", P, n_pad, U, 2, max_n, Th, pos0, xs_base, h_frame0, &win)) return WNB_ERR_INVALID;
  p.pos0 = win.pos0; p.i0 = win.i0; p.i_last = win.i_last; p.h_last = win.h_last; p.stride_xs = win.stride_xs;
  p.xs = shift_ptr(xs, -(long long)xs_base); p.h = shift_ptr(h, -(long long)h_frame0);
  p.uniforms = shift_ptr(uniforms, -(long long)win.i0); p.logits_out = shift_ptr(logits_out, -(long long)win.i0 * Q);
  p.timing = g_decode_timing;
  long long off = 0;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(host_dilations[l] >= 1 && (host_dilations[l] & (host_dilations[l] - 1)) == 0,
                "decode_warp: dilations must be powers of two");
    p.dil[l] = host_dilations[l];
    p.qoff[l] = off;
    off += (long long)host_dilations[l] * dw::kR;
  }
  p.q_per_utt = off;
  int rc = decode_warp_launch(p, W, CL, (cudaStream_t)stream_handle);
  if (rc == WNB_ERR_UNSUPPORTED) set_error("decode_warp: not enough shared memory for this depth");
  return rc;
}

}  // extern "C"
