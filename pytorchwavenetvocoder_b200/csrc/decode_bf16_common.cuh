// decode_bf16_common.cuh -- what the bf16 decoder (decode_bf16.cu) and its parallel warm-up (decode_bf16_prefill.cu)
// share: the activation tile layout, the consumer side of the weight ring, the wgmma product over ring stages, the
// packed weight stream's sizes and the cluster split of a batch.  The warm-up is bit-identical to the decoder's
// sequential warm-up only because both issue these same instructions on the same operands in the same K order.
#pragma once
#include "common.cuh"
#include "tc_ptx.cuh"

namespace wnb {
namespace db {

constexpr int kCL = 8;                    // CTAs per cluster (the portable maximum); output slices of a product
constexpr int kM = 64;                    // rows of a product (wgmma M): utterances in the decoder, positions in the prefill
constexpr int kQ = 256;
constexpr int kQc = kQ / kCL;             // classes per CTA (post-2 N)
constexpr int kTile = kM * 64 * 2;        // one [64 rows][64 ch] bf16 tile: 8 KB
constexpr int kCons = 128;                // one consumer warpgroup

// byte offset of (row, k < 64) in a [64 rows][64] bf16 tile with the 128B swizzle; of (row, channel) in a buffer of tiles
__device__ __forceinline__ uint32_t tile_off(int row, int k) {
  return (uint32_t)(row * 128 + ((((k >> 3) ^ row) & 7) << 4) + ((k & 7) << 1));
}
__device__ __forceinline__ uint32_t act_off(int row, int ch) { return (uint32_t)((ch >> 6) * kTile) + tile_off(row, ch & 63); }

__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_b32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kCons) : "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem), "l"(gmem), "r"(bytes), "r"(ptx::smem_u32(bar)) : "memory");
}

// consumer side of the weight ring: stage `st` of phase parity `ph`; a stage is released (one arrive per warp) once the
// wgmma group that read it has completed
struct Ring {
  uint32_t base; uint64_t* full; uint64_t* empty; int n; int bytes; int st; uint32_t ph; int prev;
  __device__ __forceinline__ uint32_t wait() {
    ptx::mbar_wait(&full[st], ph);
    return base + (uint32_t)(st * bytes);
  }
  __device__ __forceinline__ void release(int s, int lane) {
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  }
  // after the wgmma group of the current stage was committed: wait for it (M = 64 products are short; the producer keeps
  // the other stages streaming meanwhile), then hand the previous stage back
  __device__ __forceinline__ void committed(int lane) {
    ptx::wg_wait<0>();
    if (prev >= 0) release(prev, lane);
    prev = st;
    if (++st == n) { st = 0; ph ^= 1u; }
  }
};
// a copy of v the compiler cannot see through: keeps per-thread address arithmetic inside the step / layer loops
// instead of hoisting dozens of loop-invariant offsets into registers for the whole kernel
__device__ __forceinline__ int opaque(int v) {
  asm volatile("mov.b32 %0, %0;" : "+r"(v));
  return v;
}

// one [64 x 64] A tile times one [N x 64] B tile, accumulated into d: 4 k16 steps, A fragments from shared memory
template <int N>
__device__ __forceinline__ void mma_tile(float (&d)[N / 2], uint32_t (&a)[4][4], uint32_t a_tile, uint32_t b_tile, int fr,
                                         int fk) {
#pragma unroll
  for (int s = 0; s < 4; s++)
#pragma unroll
    for (int h = 0; h < 4; h++) a[s][h] = ld_shared_b32(a_tile + tile_off(fr + 8 * (h & 1), 16 * s + fk + 8 * (h >> 1)));
  ptx::wg_fence();
#pragma unroll
  for (int s = 0; s < 4; s++) ptx::wgmma_rs_bf16<N>(d, a[s], ptx::gmma_desc_k_sw128(b_tile + 32 * s), 1);
  ptx::wg_commit();
}

// d = sum over nch ring stages of A(c) x B(stage c); `pre(c)` runs before chunk c waits for its stage.  Returns the
// shared-memory address of the last stage, which is NOT released yet (its bias tail is still to be read).
template <int N, class ATile, class Pre>
__device__ __forceinline__ uint32_t product(float (&d)[N / 2], Ring& rg, int nch, ATile atile, Pre pre, int fr, int fk,
                                            int lane) {
#pragma unroll
  for (int i = 0; i < N / 2; i++) d[i] = 0.f;
  uint32_t a[4][4];
  uint32_t last = 0;
#pragma unroll 1
  for (int c = 0; c < nch; c++) {
    pre(c);
    last = rg.wait();
    mma_tile<N>(d, a, atile(c, last), last, fr, fk);
    rg.committed(lane);
  }
  ptx::wg_touch(d);
  return last;
}

}  // namespace db

// ---- host side: the packed per-CTA weight stream and the cluster split ----------------------------------------------
static inline int db_aux_k(int Ap) { return (Ap + 63) / 64 * 64; }
// bytes of one layer of one CTA's stream: gate chunks + b1, then res+skip chunks + b2
static inline size_t db_gate_bytes(int Ap, int R, int ks) {
  const size_t NG = R / 4;
  return NG * ((size_t)db_aux_k(Ap) + (size_t)ks * R) * 2 + NG * 4;
}
static inline size_t db_cta_bytes(int Ap, int R, int S, int ks) {
  const size_t NR = R / 8 + S / 8;
  return db_gate_bytes(Ap, R, ks) + NR * (size_t)R * 2 + NR * 4;   // per layer; the post tail is added by the callers
}
static inline size_t db_post_bytes(int S) { return (size_t)(S / 8) * S * 2 + (S / 8) * 4 + (size_t)db::kQc * S * 2 + db::kQc * 4; }
// B utterances run as ncl = ceil(B / 64) clusters of bc = ceil(B / ncl) (the last one may have fewer): cluster cl holds
// utterances cl bc .. in rows 0 .., and a row past its utterances repeats the cluster's last utterance
static inline void db_split(int B, int* ncl, int* bc) {
  *ncl = cdiv(B, db::kM);
  *bc = cdiv(B, *ncl);
}

}  // namespace wnb
