// gemm_nt_tc.cu -- tensor-core GEMM over channels-last activations:
//     D[t][n] = epi( sum_seg sum_k A_seg[t + shift_seg][k] * W_seg[n][k] )          n < N <= 256 per tile
// A rows are time steps (K-major operand straight from the (B,T,C) tensor, TMA zero fill outside [0,T) =
// causal / anti-causal padding), W is a row-major [N][K] weight matrix (K-major operand).  Hopper wgmma
// m64nNk8 tf32, fp32 accumulate in registers.  A CTA has one producer warpgroup and two consumer warpgroups and works on
// pairs of consecutive 64-row time tiles (flattened over the batch) of one column block: one producer thread streams,
// per stage of an mbarrier ring, the two tiles' [64 x 32] activation boxes and ONE [N x 32] weight box with TMA, and each
// consumer warpgroup multiplies its own activation box by the shared weight box.  So a weight box is pulled from L2 once
// per 128 time rows.  A pair whose second tile lies past the last one leaves that warpgroup with nothing but releasing
// the stages.  setmaxnreg gives the consumers 232 registers (N = 256: 128 accumulator registers) and the producer 40.
// bf16 operands (W = __nv_bfloat16): the weights arrive as bf16 [N x 32] boxes (a bf16 copy made by the caller, 64B
// swizzle); the activation box is still fp32, and the consumers read two adjacent k per shared-memory load, round them
// to bf16 (cvt.rn.bf16x2) into the register A fragment of wgmma m64nNk16 (bf16, fp32 accumulate).  The epilogues are
// the same: the accumulator is fp32 either way.
// Epilogue, straight from the accumulator registers: in the m64nN fragment a thread holds rows 16 w + lane/4 (+ 8) and
// column pairs 8 j + 2 (lane % 4) (+ 1), so the tanh partner of gate column c (c + GC) and the dz partial (c + 2 GC) sit
// in the same thread.  + bias, + residual, ReLU, * (mask > 0), or the gate forward / backward, then each warp writes its
// 16 rows x 32 columns into a swizzled staging box and one lane issues a TMA store or TMA reduce-add (.add.f32) into the
// (B,T,N) output.  The epilogue operand read from memory per tile (the gate backward's dz, the residual added to the
// plain epilogue when it is at most 64 columns wide) is loaded by TMA into a buffer per warpgroup when the tile's
// mainloop starts, so its latency hides behind the MMAs; rows past T come back as zero fill.  Bias and mask are read
// with __ldg.  The kernel is instantiated per (N, epilogue kind, operand type) so each variant gets its own register
// allocation.  Column blocks (work items ordered block-fastest so the A tiles are shared through L2), split output and
// programmatic dependent launch as options.
// Thread-block clusters (Params::cm = CM in {1, 2, 4} CTAs along x; 1 unless forced, see pick_cm for the measurements):
// the CTAs of a cluster take CM consecutive tile pairs of the same column block, and each weight box is read from L2
// once per cluster: CTA r loads rows [r N/CM, (r+1) N/CM) of it (of each half, for the gate's two half boxes) and
// multicasts them into the same ring offset of every CTA.  A stage is refilled only when the consumers of both
// warpgroups of every CTA have released it (one arrive per consumer warp on each CTA's empty barrier).  A CTA whose
// pair lies past the last one still loads its weight slice and releases the stages, without MMAs or stores.  Each
// tile's arithmetic is the same for every CM.
// Used for: the post network forward (wavenet.py:518-523) and backward, the hoisted skip GEMMs, the gate backward,
// the residual-stream data gradient dX (two time-shifted segments) with the aux gradient dhaux (reduce-add).
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_bf16.h>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>

#include "common.cuh"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace wnb {
namespace nt {

constexpr int kTM = 64;                  // time rows per tile (wgmma M)
constexpr int kASub = kTM * 32 * 4;      // 8 KB: one tile's activation box of a stage
constexpr int kStgRows = 16;             // rows of a staging box: one warp's share of the fragment
constexpr int kStg = kStgRows * 32 * 4;  // 2 KB
constexpr int kStgBytes = 8 * 2 * kStg;  // 8 consumer warps x 2 staging boxes
constexpr int kEopBox = kTM * 32 * 4;    // 8 KB: [64 x 32] box of the epilogue operand
constexpr int kMaxEop = 2;               // epilogue operand boxes per warpgroup (64 columns)
constexpr int kWG = 128;
constexpr int kConsumers = 2 * kWG;      // two warpgroups: MMA + epilogue, one tile each
constexpr int kThreadsN = kConsumers + kWG;   // + the producer warpgroup (one thread issues TMA)
constexpr int kMaxSeg = 4;

struct Seg { int amap; int shift; int K; int bmap; int b_k0; int b_n0; int b_n1; };   // b_n1 >= 0: rows of the 2nd half of N
struct alignas(64) Params {
  CUtensorMap maps[11];   // [0..3] A tensors, [4..7] weight matrices, [8] output, [9] second output, [10] epilogue operand
  Seg seg[kMaxSeg];
  int nseg, N, T, B, nstages;
  const float* bias; const float* mask; int ldmask; const float* add; int ldadd;
  int relu_out, accumulate;
  // gate epilogues (N == 128 = [64 sigmoid pre | 64 tanh pre] of gate channels gate_c0 .. gate_c0+63 of gate_R):
  //   forward  (gate_mode 1): z -> maps[8] at column gate_c0 + c
  //   backward (gate_mode 2): dz (B,T,gate_R) in;  z -> maps[8];  dpre -> maps[9] at columns gate_c0+c / gate_R+gate_c0+c
  //   backward (gate_mode 3): as 2, but N == 192 and accumulator columns 128..191 hold a partial dz (an extra GEMM
  //                           segment, e.g. dout W2res) that is added to the dz read from memory
  // bias = sigmoid-branch bias, bias2 = tanh-branch bias (already offset by gate_c0)
  const float* gate_dz; const float* bias2;
  int gate_mode, gate_c0, gate_R;
  int gate_gc;   // gate channels per tile: N == 2 * gate_gc (64, or 128 for the composed path) [+ 64 dz columns in mode 3]
  // split output: columns >= out2_col0 (> 0) are reduce-added into maps[9] at column c - out2_col0; bias / add /
  // mask / ReLU apply to the primary columns only
  int out2_col0;
  // column blocks (NtTcOpts::n_blocks), dz row pitch and z suppression of the gate-backward epilogue
  int nblk, gate_ld_dz, gate_skip_z;
  int rev;   // NtTcOpts::reverse
  int cm;    // CTAs per cluster (1, 2, 4): the weight box of a stage is multicast from CM slices of N / CM rows
  // [64 x 32] boxes of the epilogue operand (gate dz, or the plain epilogue's add) staged per tile through maps[10]
  // (0: read with __ldg)
  int neop;
};

// EPI selects the epilogue at compile time so that each variant gets its own register allocation: 0 plain (bias / add /
// ReLU / mask / split output), 1 gate forward and gate backward with z output, 2 gate backward without z (the stack path).
enum { EPI_PLAIN = 0, EPI_GATE = 1, EPI_GATE_BWD_NOZ = 2 };

// bytes of one weight row of a stage (32 k): fp32 (read as tf32) or bf16
template <typename W>
__host__ __device__ constexpr int w_row_bytes() { return std::is_same<W, __nv_bfloat16>::value ? 64 : 128; }

// W: element type of the weight operand, float (the tensor cores read it as tf32) or __nv_bfloat16
template <int N, int EPI, typename W>
__global__ void __launch_bounds__(kThreadsN, 1) gemm_nt_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kBf16 = std::is_same<W, __nv_bfloat16>::value;
  constexpr int kWRow = w_row_bytes<W>();
  constexpr int stage_bytes = 2 * kASub + N * kWRow;   // [A box tile 0 | A box tile 1 | weight box]
  unsigned char* ring = smem;
  unsigned char* stg_base = ring + (size_t)p.nstages * stage_bytes;
  unsigned char* eop_base = stg_base + kStgBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(eop_base + 2 * p.neop * kEopBox);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.nstages;
  uint64_t* eop_full = bars + 2 * p.nstages;   // [2]: one per consumer warpgroup
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_b = (p.T + kTM - 1) / kTM;
  const int ntt = p.B * tiles_per_b;   // time tiles
  const int npairs = (ntt + 1) / 2;
  // a group = CM consecutive tile pairs x one column block, column block fastest: the blocks of one pair share A via L2
  const int cm = p.cm, rank = blockIdx.x % cm, cluster = blockIdx.x / cm, nclusters = gridDim.x / cm;
  const int ngroups = (npairs + cm - 1) / cm * p.nblk;
  int kchunks = 0;
  for (int s = 0; s < p.nseg; s++) kchunks += p.seg[s].K / 32;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], (kConsumers / 32) * cm);   // one arrive per consumer warp of every CTA of the cluster
    }
    ptx::mbar_init(&eop_full[0], 1);
    ptx::mbar_init(&eop_full[1], 1);
    ptx::fence_barrier_init();
  }
  // the peers multicast into this CTA's ring and arrive on its barriers: all of them must see the initialised barriers
  if (cm > 1) ptx::cluster_sync();
  else __syncthreads();
  // programmatic dependent launch: the set-up above overlapped the previous kernel's tail; from here on this
  // kernel reads / writes memory that kernel may have produced
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp >= kConsumers / 32) {
    // =============================== TMA producer warpgroup ===============================
    ptx::setmaxnreg_dec<40>();
    if (warp == kConsumers / 32 && ptx::elect_one()) {
      for (int i = 0; i < 11; i++) ptx::prefetch_tmap(&p.maps[i]);
      const uint16_t cta_mask = (uint16_t)((1u << cm) - 1);
      // this CTA's slice of a weight box (rows wr * rank .. of each half box) -> every CTA of the cluster
      auto load_w = [&](unsigned char* box, const Seg& sg, int k, int n, int box_rows, uint64_t* bar) {
        const int wr = box_rows / cm;
        if (cm == 1) ptx::tma_load_2d(box, &p.maps[sg.bmap], bar, k, n);
        else ptx::tma_load_2d_multicast(box + rank * wr * kWRow, &p.maps[sg.bmap], bar, k, n + rank * wr, cta_mask);
      };
      uint32_t st = 0, ph = 0;
      for (int grp = cluster; grp < ngroups; grp += nclusters) {
        const int ge = p.rev ? ngroups - 1 - grp : grp;
        const int tg = ge / p.nblk, ncol0 = (ge - tg * p.nblk) * N;
        const int tt0 = 2 * (tg * cm + rank);   // the pair's first tile; the second is tt0 + 1
        const int ntiles = tt0 + 1 < ntt ? 2 : (tt0 < ntt ? 1 : 0);
        int tb[2], tt[2];
#pragma unroll
        for (int h = 0; h < 2; h++) { tb[h] = (tt0 + h) / tiles_per_b; tt[h] = (tt0 + h - tb[h] * tiles_per_b) * kTM; }
        for (int s = 0; s < p.nseg; s++) {
          const Seg sg = p.seg[s];
          for (int kc = 0; kc < sg.K / 32; kc++) {
            ptx::mbar_wait<ptx::kStoreFault>(&empty[st], ph ^ 1);
            ptx::mbar_arrive_expect_tx(&full[st], stage_bytes - (2 - ntiles) * kASub);
            unsigned char* dst = ring + (size_t)st * stage_bytes;
#pragma unroll
            for (int h = 0; h < 2; h++)
              if (h < ntiles) ptx::tma_load_3d(dst + h * kASub, &p.maps[sg.amap], &full[st], kc * 32, tt[h] + sg.shift, tb[h]);
            if (sg.b_n1 >= 0) {   // N = two row ranges of N/2 each (sigmoid rows, tanh rows)
              load_w(dst + 2 * kASub, sg, sg.b_k0 + kc * 32, sg.b_n0, N / 2, &full[st]);
              load_w(dst + 2 * kASub + (N / 2) * kWRow, sg, sg.b_k0 + kc * 32, sg.b_n1, N / 2, &full[st]);
            } else {
              load_w(dst + 2 * kASub, sg, sg.b_k0 + kc * 32, sg.b_n0 + ncol0, N, &full[st]);
            }
            if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
          }
        }
      }
    }
    // no CTA may exit while a peer can still multicast into its ring or arrive on its barriers
    __syncwarp();
    if (cm > 1) ptx::cluster_sync();
    return;
  }

  // =============================== consumer warpgroups: wgmma mainloop + epilogue ===============================
  ptx::setmaxnreg_inc<232>();
  const int wg = warp >> 2;               // warpgroup: tile wg of each pair
  const int wq = warp & 3;                // warp in the warpgroup: rows 16 wq .. 16 wq + 15 of the tile
  const int rq = lane >> 2, cq = 2 * (lane & 3);   // fragment row (+ 8) and column pair (+ 8 j) of this thread
  unsigned char* stg = stg_base + warp * 2 * kStg;
  unsigned char* eop = eop_base + wg * p.neop * kEopBox;
  const uint32_t ring_u32 = ptx::smem_u32(ring);
  uint32_t st = 0, ph = 0, nstore = 0, eph = 0;
  // stage s may be refilled as far as this warp is concerned: one arrive on the empty barrier of every CTA of the cluster
  auto release = [&](uint32_t s) {
    __syncwarp();
    if (lane == 0) {
      if (cm == 1) ptx::mbar_arrive(&empty[s]);
      else
        for (int r = 0; r < cm; r++) ptx::mbar_arrive_cluster(&empty[s], (uint32_t)r);
    }
  };
  for (int grp = cluster; grp < ngroups; grp += nclusters) {
    const int ge = p.rev ? ngroups - 1 - grp : grp;
    const int tg = ge / p.nblk, ncol0 = (ge - tg * p.nblk) * N;
    const int tt = 2 * (tg * cm + rank) + wg;
    const int b = tt / tiles_per_b, t0 = (tt - b * tiles_per_b) * kTM;
    if (tt >= ntt) {   // past the last tile (partial last pair or group): only keep the stages moving
      for (int kc = 0; kc < kchunks; kc++) {
        ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
        release(st);
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      }
      continue;
    }
    if (p.neop) {
      // this tile's epilogue operand -> the warpgroup's buffer, once every warp is done reading the previous tile's
      ptx::named_bar(1 + wg, kWG);
      if (wq == 0 && lane == 0) {
        const int c0 = p.gate_mode ? p.gate_c0 : ncol0;
        ptx::mbar_arrive_expect_tx(&eop_full[wg], p.neop * kEopBox);
        for (int k = 0; k < p.neop; k++) ptx::tma_load_3d(eop + k * kEopBox, &p.maps[10], &eop_full[wg], c0 + 32 * k, t0, b);
      }
    }
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[i] = 0.f;
    uint32_t prev = 0xFFFFFFFFu;
    if constexpr (!kBf16) {
      for (int kc = 0; kc < kchunks; kc++) {
        ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
        ptx::wg_fence();
        const uint32_t a_addr = ring_u32 + st * stage_bytes + wg * kASub, b_addr = ring_u32 + st * stage_bytes + 2 * kASub;
#pragma unroll
        for (int k = 0; k < 4; k++)
          ptx::wgmma_ss<N>(d, ptx::gmma_desc_k_sw128(a_addr + 32 * k), ptx::gmma_desc_k_sw128(b_addr + 32 * k), 1);
        ptx::wg_commit();
        ptx::wg_wait<1>();                   // the previous chunk's MMAs are done: its stage can be refilled
        if (prev != 0xFFFFFFFFu) release(prev);
        prev = st;
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      }
    } else {
      // A fragments (rows 16 wq + lane/4 (+ 8), k pairs 2 (lane % 4) (+ 8)) converted from the fp32 box into one of two
      // register sets: wgmma reads them asynchronously, so a set is refilled only after the chunk that used it is done
      const int fr = 16 * wq + rq, fk = cq;
      uint32_t a0[2][4], a1[2][4];
      auto chunk = [&](uint32_t (&a)[2][4]) {
        ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
        const unsigned char* as = ring + (size_t)st * stage_bytes + wg * kASub;
#pragma unroll
        for (int k = 0; k < 2; k++)
#pragma unroll
          for (int h = 0; h < 4; h++) {
            const float2 v = *reinterpret_cast<const float2*>(as + ptx::sw128_off(fr + 8 * (h & 1), 16 * k + fk + 8 * (h >> 1)));
            a[k][h] = ptx::cvt_bf16x2(v.x, v.y);
          }
        ptx::wg_fence();
        const uint32_t b_addr = ring_u32 + st * stage_bytes + 2 * kASub;
#pragma unroll
        for (int k = 0; k < 2; k++) ptx::wgmma_rs_bf16<N>(d, a[k], ptx::gmma_desc_k_sw64(b_addr + 32 * k), 1);
        ptx::wg_commit();
        ptx::wg_wait<1>();                 // the previous chunk's MMAs are done: its stage can be refilled
        if (prev != 0xFFFFFFFFu) release(prev);
        prev = st;
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      };
      for (int kc = 0; kc < kchunks; kc += 2) {
        chunk(a0);
        if (kc + 1 < kchunks) chunk(a1);
      }
    }
    ptx::wg_wait<0>();
    ptx::wg_touch(d);
    if (prev != 0xFFFFFFFFu) release(prev);

    // ---- epilogue from registers.  Value v[4 jj + 2 h + e] of a 32-column chunk cb is accumulator d[4 (4 cb + jj) + 2 h
    //      + e]: row rq + 8 h of this warp's 16, column 32 cb + 8 jj + cq + e ----
    const int r16 = 16 * wq;
    bool row_ok[2];
    size_t grow[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int t = t0 + r16 + rq + 8 * h;
      row_ok[h] = t < p.T;
      grow[h] = (size_t)b * p.T + (row_ok[h] ? t : 0);
    }
    if (p.neop) {
      ptx::mbar_wait<ptx::kStoreFault>(&eop_full[wg], eph);
      eph ^= 1;
    }
    // two values of the epilogue operand at row rq + 8 h, column c (even): from the staged boxes, or from memory
    auto operand = [&](const float* g, int ld, int col0, int c, int h) -> float2 {
      if (p.neop) return *reinterpret_cast<const float2*>(eop + (c >> 5) * kEopBox + ptx::sw128_off(r16 + rq + 8 * h, c & 31));
      return row_ok[h] ? __ldg(reinterpret_cast<const float2*>(g + grow[h] * ld + col0 + c)) : make_float2(0.f, 0.f);
    };
    // 16 values -> this warp's next staging box -> TMA store (or reduce-add) of [16 rows x 32 columns] at column col
    auto store16 = [&](const float (&v)[16], const CUtensorMap* map, int col, bool reduce) {
      unsigned char* sb = stg + (nstore & 1) * kStg;
      if (lane == 0) ptx::bulk_wait_read<1>();
      __syncwarp();
#pragma unroll
      for (int jj = 0; jj < 4; jj++)
#pragma unroll
        for (int h = 0; h < 2; h++)
          *reinterpret_cast<float2*>(sb + ptx::sw128_off(rq + 8 * h, 8 * jj + cq)) = make_float2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
      ptx::fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        if (reduce) ptx::tma_reduce_add_3d(map, sb, col, t0 + r16, b);
        else ptx::tma_store_3d(map, sb, col, t0 + r16, b);
        ptx::bulk_commit();
      }
      nstore++;
    };
    if constexpr (EPI == EPI_GATE_BWD_NOZ || EPI == EPI_GATE) {
      // ---- gate epilogues: sigmoid column c pairs with tanh column GC + c (d[i + GC/2]) and, in mode 3, the dz
      //      partial at 2 GC + c (d[i + GC]); GC = 64, or 128 at N = 256.  Other N never take a gate epilogue. ----
      if constexpr (N == 128 || N == 192 || N == 256) {
        constexpr int GC = N == 256 ? 128 : 64;
        const bool bwd = p.gate_mode >= 2;
#pragma unroll
        for (int cb = 0; cb < GC / 32; cb++) {
          float a[16], g[16], z[16];
#pragma unroll
          for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
              const int c = 32 * cb + 8 * jj + cq, v = 4 * jj + 2 * h, i = 4 * (4 * cb + jj) + 2 * h;
              float2 dz2 = make_float2(0.f, 0.f);
              if (bwd) dz2 = operand(p.gate_dz, p.gate_ld_dz, p.gate_c0, c, h);
              const float dzs[2] = {dz2.x, dz2.y};
              const float bsa[2] = {__ldg(p.bias + c), __ldg(p.bias + c + 1)};
              const float bta[2] = {__ldg(p.bias2 + c), __ldg(p.bias2 + c + 1)};
#pragma unroll
              for (int e = 0; e < 2; e++) {
                const float sg = 0.5f * ptx::tanh_approx(0.5f * (d[i + e] + bsa[e])) + 0.5f;
                const float th = ptx::tanh_approx(d[i + e + GC / 2] + bta[e]);
                if (!bwd) { z[v + e] = sg * th; continue; }   // forward: z only
                float dz = dzs[e];
                if constexpr (N == 192)
                  if (p.gate_mode == 3) dz += d[i + e + GC];
                a[v + e] = dz * th * sg * (1.f - sg);      // d pre-sigmoid
                g[v + e] = dz * sg * (1.f - th * th);      // d pre-tanh
                z[v + e] = sg * th;                        // z
              }
            }
          const int col = p.gate_c0 + 32 * cb;
          if (EPI == EPI_GATE && !(bwd && p.gate_skip_z)) store16(z, &p.maps[8], col, false);
          if (bwd) {
            store16(a, &p.maps[9], col, false);
            store16(g, &p.maps[9], p.gate_R + col, false);
          }
        }
      }
    }
    if constexpr (EPI == EPI_PLAIN) {
#pragma unroll
      for (int cb = 0; cb < N / 32; cb++) {
        const int c0 = 32 * cb;
        const bool second = p.out2_col0 > 0 && c0 >= p.out2_col0;
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; i++) v[i] = d[16 * cb + i];
        if (p.bias && !second) {
#pragma unroll
          for (int jj = 0; jj < 4; jj++) {
            const float b0 = __ldg(p.bias + ncol0 + c0 + 8 * jj + cq), b1 = __ldg(p.bias + ncol0 + c0 + 8 * jj + cq + 1);
#pragma unroll
            for (int h = 0; h < 2; h++) { v[4 * jj + 2 * h] += b0; v[4 * jj + 2 * h + 1] += b1; }
          }
        }
        if (p.add && !second) {
#pragma unroll
          for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int h = 0; h < 2; h++)
              if (p.neop || row_ok[h]) {
                const float2 a = operand(p.add, p.ldadd, ncol0, c0 + 8 * jj + cq, h);
                v[4 * jj + 2 * h] += a.x; v[4 * jj + 2 * h + 1] += a.y;
              }
        }
        if (p.relu_out && !second) {
#pragma unroll
          for (int i = 0; i < 16; i++) v[i] = fmaxf(v[i], 0.f);
        }
        if (p.mask && !second) {
#pragma unroll
          for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int h = 0; h < 2; h++)
              if (row_ok[h]) {
                const float2 m = __ldg(reinterpret_cast<const float2*>(p.mask + grow[h] * p.ldmask + ncol0 + c0 + 8 * jj + cq));
                v[4 * jj + 2 * h] = m.x > 0.f ? v[4 * jj + 2 * h] : 0.f;
                v[4 * jj + 2 * h + 1] = m.y > 0.f ? v[4 * jj + 2 * h + 1] : 0.f;
              }
        }
        if (second) store16(v, &p.maps[9], c0 - p.out2_col0, true);
        else store16(v, &p.maps[8], ncol0 + c0, p.accumulate != 0);
      }
    }
  }
  if (lane == 0) ptx::bulk_wait<0>();
  __syncwarp();
  if (cm > 1) ptx::cluster_sync();
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}
static bool map3(CUtensorMap* m, const float* base, int C, int T, int B, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B};
  cuuint64_t gstr[2] = {(cuuint64_t)C * 4, (cuuint64_t)C * 4 * (cuuint64_t)T};
  cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1}, es[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static bool map2(CUtensorMap* m, const float* base, int K, int Nrows, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)Nrows};
  cuuint64_t gstr[1] = {(cuuint64_t)K * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows}, es[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// the bf16 weight matrix: [box_rows x 32] boxes of 64-byte rows, 64B swizzle (the layout gmma_desc_k_sw64 describes)
static bool map2_bf16(CUtensorMap* m, const __nv_bfloat16* base, int K, int Nrows, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)Nrows};
  cuuint64_t gstr[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows}, es[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(base), gdim, gstr, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Clusters of cm CTAs of `kernel` that can be resident at once on the current device (a cluster lives in one GPC, so this
// can be less than SMs x CTAs per SM / cm), cached per (device, kernel, shared memory, cm); 0 if the query fails.
template <typename K>
static int max_active_clusters(K kernel, size_t smem, int cm) {
  static std::mutex mu;
  static std::map<std::tuple<int, const void*, size_t, int>, int> fit;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  const auto key = std::make_tuple(dev, reinterpret_cast<const void*>(kernel), smem, cm);
  std::lock_guard<std::mutex> lk(mu);
  auto it = fit.find(key);
  if (it != fit.end()) return it->second;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cm);
  cfg.blockDim = dim3(kThreadsN);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cm;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) n = 0;
  return fit[key] = n;
}

// ngroups: cluster work items (p.cm tile pairs x one column block).  One CTA per SM: its three warpgroups take the whole
// register file (setmaxnreg 40 / 232 / 232) and most of the shared memory.
template <int N, int EPI, typename W>
static cudaError_t launch_n(int ngroups, size_t smem, cudaStream_t st, const Params& p) {
  cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(gemm_nt_tc_kernel<N, EPI, W>), smem);
  if (e != cudaSuccess) return e;
  int slots = device_sms();
  if (p.cm > 1) {
    slots = max_active_clusters(gemm_nt_tc_kernel<N, EPI, W>, smem, p.cm);
    if (slots < 1) return cudaErrorInvalidConfiguration;
  }
  const int grid = (ngroups < slots ? ngroups : slots) * p.cm;
  return launch_pdl(gemm_nt_tc_kernel<N, EPI, W>, grid, kThreadsN, smem, st, p.cm, p);
}

template <int EPI, typename W>
static cudaError_t launch_epi(int N, int ngroups, size_t smem, cudaStream_t st, const Params& p) {
  switch (N) {
    case 32: return launch_n<32, EPI, W>(ngroups, smem, st, p);
    case 64: return launch_n<64, EPI, W>(ngroups, smem, st, p);
    case 96: return launch_n<96, EPI, W>(ngroups, smem, st, p);
    case 128: return launch_n<128, EPI, W>(ngroups, smem, st, p);
    case 160: return launch_n<160, EPI, W>(ngroups, smem, st, p);
    case 192: return launch_n<192, EPI, W>(ngroups, smem, st, p);
    case 224: return launch_n<224, EPI, W>(ngroups, smem, st, p);
    default: return launch_n<256, EPI, W>(ngroups, smem, st, p);
  }
}

// CTAs per cluster for a launch whose weight boxes have box_rows rows (each half box, for the gate's two).
// The default is 1 for every launch.  Measured on an H100 80GB HBM3 (power limit not reported), bench.py's step
// (8 x 23 040, ms per step for the kind, CM = 1 / 2 / 4): skip GEMM 1.94 / 2.19 / 2.40, dZ_all 1.84 / 1.78 / 2.10, gate backward 4.62 / 4.77 /
// 5.24, dx 3.97 / 4.28 / 4.68; whole step 24.9 / 25.5 / 27.2 ms (one consumer warpgroup per CTA).  With two consumer
// warpgroups sharing each weight box, once on the same kind of card (CM = 1 / 2): skip GEMM 1.01 / 1.04, dZ_all 1.21 /
// 1.24, gate backward 3.53 / 3.64, dx 2.74 / 2.78; step 20.53 / 20.76 ms.  Halving the weight bytes pulled from L2 again
// does not pay for the cluster-wide coupling of the ring.
// WNB_NT_CLUSTER=1, 2 or 4 in the environment forces CM (tests, A/B timing); it is read on every call.  Either way CM is
// halved until each CTA's slice of a box is a whole number of 8-row swizzle atoms (1024 B tf32, 512 B bf16), the
// alignment at which a slice lands in the same swizzled layout as the whole box.
static int pick_cm(int box_rows) {
  const char* e = getenv("WNB_NT_CLUSTER");
  int cm = 1;
  if (e && (e[0] == '1' || e[0] == '2' || e[0] == '4') && e[1] == 0) cm = e[0] - '0';
  while (cm > 1 && box_rows % (8 * cm) != 0) cm /= 2;
  return cm;
}

}  // namespace nt

int gemm_nt_tc(const NtTcSeg* segs, int nseg, int N, float* out, int ld_out, const float* bias, const float* mask,
               int ldmask, const float* add, int ldadd, int relu_out, int accumulate, int B, int T, cudaStream_t st,
               const float* gate_dz, float* gate_dpre, float* out2, int ld_out2, int out2_col0, const NtTcGate* gate,
               const NtTcOpts* opts) {
  using namespace nt;
  if (nseg < 1 || nseg > kMaxSeg || N % 32 != 0 || N < 32 || N > 512 || (N > 256 && N != 512) || ld_out % 4 != 0) {
    set_error("gemm_nt_tc: unsupported shape (nseg=%d N=%d)", nseg, N);
    return WNB_ERR_INVALID;
  }
  Params p;
  memset(&p, 0, sizeof(p));
  p.nblk = (opts && opts->n_blocks > 1) ? opts->n_blocks : 1;
  if (N == 512) {   // the accumulator of one tile is at most 256 columns: two column blocks
    if (gate || gate_dz || out2 || p.nblk > 1) {
      set_error("gemm_nt_tc: N = 512 is for plain epilogues without column blocks");
      return WNB_ERR_INVALID;
    }
    N = 256;
    p.nblk = 2;
  }
  const int nbox = gate ? N / 2 : N;   // (gate: two boxes of GC = N/2 rows, sigmoid rows and tanh rows)
  p.cm = pick_cm(nbox);                // (each CTA of a cluster loads nbox / cm rows of each box)
  const bool bf16 = segs[0].wb != nullptr;
  for (int s = 0; s < nseg; s++) {
    if (segs[s].K % 32 != 0) { set_error("gemm_nt_tc: K must be a multiple of 32"); return WNB_ERR_INVALID; }
    if ((segs[s].wb != nullptr) != bf16) {
      set_error("gemm_nt_tc: either every segment or none has a bf16 weight copy");
      return WNB_ERR_INVALID;
    }
    if (bf16 && (segs[s].w_cols % 8 != 0 || (reinterpret_cast<uintptr_t>(segs[s].wb) & 15))) {
      set_error("gemm_nt_tc: a bf16 weight matrix needs a row pitch of 8k elements and a 16-byte aligned base");
      return WNB_ERR_INVALID;
    }
    if (!map3(&p.maps[s], segs[s].a, segs[s].CA, T, B, kTM) ||
        !(bf16 ? map2_bf16(&p.maps[4 + s], segs[s].wb, segs[s].w_cols, segs[s].w_rows, nbox / p.cm)
               : map2(&p.maps[4 + s], segs[s].w, segs[s].w_cols, segs[s].w_rows, nbox / p.cm))) {
      set_error("gemm_nt_tc: tensor map creation failed");
      return WNB_ERR_CUDA;
    }
    p.seg[s] = Seg{s, segs[s].shift, segs[s].K, 4 + s, segs[s].k0, segs[s].n0, -1};
  }
  for (int s = nseg; s < 4; s++) { p.maps[s] = p.maps[0]; p.maps[4 + s] = p.maps[4]; }
  if (!map3(&p.maps[8], out, ld_out, T, B, kStgRows)) { set_error("gemm_nt_tc: output map failed"); return WNB_ERR_CUDA; }
  p.maps[9] = p.maps[8];
  if (gate_dz) {   // R = 64 shorthand used by the fused-shape backward: whole gate in one launch
    const bool fused_dz = opts && opts->gate_fused_dz;
    if (N != (fused_dz ? 192 : 128) || !gate_dpre || !bias || !map3(&p.maps[9], gate_dpre, 128, T, B, kStgRows)) {
      set_error("gemm_nt_tc: bad gate-backward configuration");
      return WNB_ERR_INVALID;
    }
    if (reinterpret_cast<uintptr_t>(bias) & 15) { set_error("gemm_nt_tc: gate bias must be 16-byte aligned"); return WNB_ERR_INVALID; }
    p.gate_dz = gate_dz; p.bias = bias; p.bias2 = bias + 64; p.gate_mode = fused_dz ? 3 : 2; p.gate_c0 = 0; p.gate_R = 64;
    p.gate_gc = 64;
  }
  if (gate) {      // general form: GC = N/2 (64 or 128) gate channels [c0, c0+GC) of R; W rows c0.. (sigmoid) and R+c0.. (tanh)
    const int GC = N / 2;
    if ((N != 128 && N != 256) || gate->R % GC != 0 || gate->c0 % GC != 0 || gate->c0 + GC > gate->R || !gate->bias_sig ||
        !gate->bias_tanh || (gate->mode != 1 && gate->mode != 2) || (gate->mode == 2 && (!gate->dz || !gate->dpre))) {
      set_error("gemm_nt_tc: bad gate configuration");
      return WNB_ERR_INVALID;
    }
    if (gate->mode == 2 && !map3(&p.maps[9], gate->dpre, 2 * gate->R, T, B, kStgRows)) {
      set_error("gemm_nt_tc: dpre map failed");
      return WNB_ERR_CUDA;
    }
    for (int s = 0; s < nseg; s++) { p.seg[s].b_n0 = gate->c0; p.seg[s].b_n1 = gate->R + gate->c0; }
    p.bias = gate->bias_sig; p.bias2 = gate->bias_tanh; p.gate_dz = gate->dz;
    p.gate_mode = gate->mode; p.gate_c0 = gate->c0; p.gate_R = gate->R; p.gate_gc = GC;
  }
  if (out2) {
    if (gate_dz || out2_col0 <= 0 || out2_col0 % 32 != 0 || out2_col0 >= N || !map3(&p.maps[9], out2, ld_out2, T, B, kStgRows)) {
      set_error("gemm_nt_tc: bad split-output configuration");
      return WNB_ERR_INVALID;
    }
    p.out2_col0 = out2_col0;
  }
  p.nseg = nseg; p.N = N; p.T = T; p.B = B;
  p.gate_ld_dz = (opts && opts->gate_ld_dz > 0) ? opts->gate_ld_dz : p.gate_R;
  p.gate_skip_z = (opts && opts->gate_skip_z) ? 1 : 0;
  if (p.nblk > 1 && (p.gate_mode || out2)) {
    set_error("gemm_nt_tc: column blocks are for plain epilogues");
    return WNB_ERR_INVALID;
  }
  if (!p.gate_mode) p.bias = bias;   // (the gate modes have already installed their own bias pointers)
  p.mask = mask; p.ldmask = ldmask; p.add = add; p.ldadd = ldadd;
  p.relu_out = relu_out; p.accumulate = accumulate;
  p.rev = (opts && opts->reverse) ? 1 : 0;
  const int epi = !p.gate_mode ? EPI_PLAIN : ((p.gate_mode >= 2 && p.gate_skip_z) ? EPI_GATE_BWD_NOZ : EPI_GATE);
  if (epi == EPI_GATE_BWD_NOZ && (p.gate_gc != 64 || (reinterpret_cast<uintptr_t>(p.gate_dz) & 15) || p.gate_ld_dz % 4)) {
    set_error("gemm_nt_tc: the gate backward without z needs 64 gate channels and a 16-byte aligned dz");
    return WNB_ERR_INVALID;
  }
  // the epilogue operand that TMA stages per tile: the gate backward's dz (64 gate channels), or the plain epilogue's
  // residual add when it is at most 64 columns wide (wider ones, e.g. the post network's, are read with __ldg).  TMA needs a
  // 16-byte aligned base and row pitch.
  auto tma_ok = [](const void* ptr, int ld) { return !(reinterpret_cast<uintptr_t>(ptr) & 15) && ld % 4 == 0; };
  const int add_cols = out2 ? out2_col0 : N;
  if (p.gate_mode >= 2 && p.gate_gc == 64 && tma_ok(p.gate_dz, p.gate_ld_dz)) {
    if (!map3(&p.maps[10], p.gate_dz, p.gate_ld_dz, T, B, kTM)) { set_error("gemm_nt_tc: dz map failed"); return WNB_ERR_CUDA; }
    p.neop = 2;
  } else if (!p.gate_mode && add && add_cols <= 32 * kMaxEop && tma_ok(add, ldadd)) {
    if (!map3(&p.maps[10], add, ldadd, T, B, kTM)) { set_error("gemm_nt_tc: add map failed"); return WNB_ERR_CUDA; }
    p.neop = add_cols / 32;
  } else {
    p.maps[10] = p.maps[8];
  }
  // shared memory: ring stages (two A boxes + weight box) | 8 warps x 2 staging boxes | 2 warpgroups x epilogue operand
  // boxes | barriers
  const int stage_bytes = 2 * kASub + N * (bf16 ? w_row_bytes<__nv_bfloat16>() : w_row_bytes<float>());
  const int fixed = kStgBytes + 2 * p.neop * kEopBox + 1024 + 256;
  int nst = (227 * 1024 - fixed) / stage_bytes;
  if (nst > 6) nst = 6;
  if (nst < 2) { set_error("gemm_nt_tc: N too large"); return WNB_ERR_INVALID; }
  p.nstages = nst;
  const size_t smem = (size_t)fixed + (size_t)nst * stage_bytes;
  const int ngroups = cdiv(cdiv(B * cdiv(T, kTM), 2), p.cm) * p.nblk;
  cudaError_t le;
  if (bf16) {   // (the gate backward without z belongs to the tf32 stack only)
    if (epi == EPI_PLAIN) le = launch_epi<EPI_PLAIN, __nv_bfloat16>(N, ngroups, smem, st, p);
    else if (epi == EPI_GATE) le = launch_epi<EPI_GATE, __nv_bfloat16>(N, ngroups, smem, st, p);
    else { set_error("gemm_nt_tc: no bf16 variant of the gate backward without z"); return WNB_ERR_INVALID; }
  } else if (epi == EPI_PLAIN) le = launch_epi<EPI_PLAIN, float>(N, ngroups, smem, st, p);
  else if (epi == EPI_GATE) le = launch_epi<EPI_GATE, float>(N, ngroups, smem, st, p);
  else le = launch_epi<EPI_GATE_BWD_NOZ, float>(N, ngroups, smem, st, p);
  if (le != cudaSuccess) { set_error("gemm_nt_tc: launch failed: %s", cudaGetErrorString(le)); return WNB_ERR_CUDA; }
  WNB_CHECK_LAUNCH("gemm_nt_tc");
  return WNB_OK;
}

}  // namespace wnb
