// gemm_nt_tc.cu -- tensor-core GEMM over channels-last activations:
//     D[t][n] = epi( sum_seg sum_k A_seg[t + shift_seg][k] * W_seg[n][k] )          n < N <= 256 per tile
// A rows are time steps (K-major operand straight from the (B,T,C) tensor, TMA zero fill outside [0,T) =
// causal / anti-causal padding), W is a row-major [N][K] weight matrix (K-major operand).  Hopper wgmma
// m64nNk8 tf32, fp32 accumulate in registers of one consumer warpgroup; one producer warp streams
// [64 x 32] activation boxes and [N x 32] weight boxes through an mbarrier ring with TMA.
// bf16 operands (W = __nv_bfloat16): the weights arrive as bf16 [N x 32] boxes (a bf16 copy made by the caller, 64B
// swizzle); the activation box is still fp32, and the consumers read two adjacent k per shared-memory load, round them
// to bf16 (cvt.rn.bf16x2) into the register A fragment of wgmma m64nNk16 (bf16, fp32 accumulate).  The epilogues are
// the same: the accumulator is fp32 either way.
// Epilogue: the accumulator is written to shared memory column-major, then each consumer thread owns one time row
// and 32-column chunks (warp w: rows 32 (w & 1) .., chunks w >> 1, (w >> 1) + 2, ...): + bias, ReLU, * (mask > 0),
// + residual, then a swizzled per-warp staging box and a TMA store or TMA reduce-add (.add.f32) into the (B,T,N)
// output; gate forward / backward epilogues for the residual blocks.  The kernel is instantiated per (N, epilogue
// kind) so each variant gets its own register allocation.  Column blocks (tiles ordered block-fastest so the A tile
// is shared through L2), split output and programmatic dependent launch as options.
// Thread-block clusters (Params::cm = CM in {1, 2, 4} CTAs along x; 1 unless forced, see pick_cm for the measurements):
// the CTAs of a cluster take CM consecutive time tiles (flattened over the batch) of the same column block, and each
// weight box is read from L2 once per cluster: CTA r loads rows [r N/CM, (r+1) N/CM) of it (of each half, for the gate's
// two half boxes) and multicasts them into the same ring offset of every CTA.  A stage is refilled only when the
// consumers of every CTA have released it (one arrive per consumer warp on each CTA's empty barrier).  A CTA whose tile
// lies past the last one still loads its weight slice and releases the stages, without MMAs or stores.  Each tile's
// arithmetic is the same for every CM.
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
constexpr int kASub = kTM * 32 * 4;      // 8 KB
constexpr int kStg = 32 * 32 * 4;        // 4 KB
constexpr int kConsumers = 128;          // one warpgroup: MMA + epilogue
constexpr int kThreadsN = kConsumers + 32;
constexpr int kAccLd = kTM + 4;          // column pitch (floats) of the shared-memory accumulator: conflict-free both ways
// bytes of the accumulator copy, rounded up so that the staging boxes behind it keep the 1024-byte alignment the
// 128B-swizzled TMA stores need
__host__ __device__ constexpr int acc_bytes(int N) { return (N * kAccLd * 4 + 1023) & ~1023; }
constexpr int kMaxSeg = 4;

struct Seg { int amap; int shift; int K; int bmap; int b_k0; int b_n0; int b_n1; };   // b_n1 >= 0: rows of the 2nd half of N
struct alignas(64) Params {
  CUtensorMap maps[10];   // [0..3] A tensors, [4..7] weight matrices, [8] output, [9] second output
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
};

// EPI selects the epilogue at compile time so that each variant gets its own register allocation: 0 plain (bias / add /
// ReLU / mask / split output), 1 gate forward and gate backward with z output, 2 gate backward without z (the stack path).
enum { EPI_PLAIN = 0, EPI_GATE = 1, EPI_GATE_BWD_NOZ = 2 };

// 16 consecutive accumulator columns of one row out of the column-major shared-memory copy
__device__ __forceinline__ void acc_ld16(const float* acc, int col, int row, float (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 16; i++) v[i] = acc[(col + i) * kAccLd + row];
}

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
  constexpr int stage_bytes = kASub + N * kWRow;
  unsigned char* ring = smem;
  float* accs = reinterpret_cast<float*>(ring + (size_t)p.nstages * stage_bytes);
  unsigned char* stg_base = reinterpret_cast<unsigned char*>(accs) + acc_bytes(N);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg_base + 4 * 2 * kStg);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.nstages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_b = (p.T + kTM - 1) / kTM;
  const int ntt = p.B * tiles_per_b;   // time tiles
  // a group = CM consecutive time tiles x one column block, column block fastest: the blocks of one time tile share A via L2
  const int cm = p.cm, rank = blockIdx.x % cm, cluster = blockIdx.x / cm, nclusters = gridDim.x / cm;
  const int ngroups = (ntt + cm - 1) / cm * p.nblk;
  int kchunks = 0;
  for (int s = 0; s < p.nseg; s++) kchunks += p.seg[s].K / 32;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], (kConsumers / 32) * cm);   // one arrive per consumer warp of every CTA of the cluster
    }
    ptx::fence_barrier_init();
  }
  // the peers multicast into this CTA's ring and arrive on its barriers: all of them must see the initialised barriers
  if (cm > 1) ptx::cluster_sync();
  else __syncthreads();
  // programmatic dependent launch: the set-up above overlapped the previous kernel's tail; from here on this
  // kernel reads / writes memory that kernel may have produced
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp == 4) {
    // =============================== TMA producer ===============================
    if (ptx::elect_one()) {
      for (int i = 0; i < 10; i++) ptx::prefetch_tmap(&p.maps[i]);
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
        const int tt = tg * cm + rank;
        const bool has_tile = tt < ntt;
        const int b = tt / tiles_per_b, t0 = (tt - b * tiles_per_b) * kTM;
        for (int s = 0; s < p.nseg; s++) {
          const Seg sg = p.seg[s];
          for (int kc = 0; kc < sg.K / 32; kc++) {
            ptx::mbar_wait(&empty[st], ph ^ 1);
            ptx::mbar_arrive_expect_tx(&full[st], has_tile ? stage_bytes : stage_bytes - kASub);
            unsigned char* dst = ring + (size_t)st * stage_bytes;
            if (has_tile) ptx::tma_load_3d(dst, &p.maps[sg.amap], &full[st], kc * 32, t0 + sg.shift, b);
            if (sg.b_n1 >= 0) {   // N = two row ranges of N/2 each (sigmoid rows, tanh rows)
              load_w(dst + kASub, sg, sg.b_k0 + kc * 32, sg.b_n0, N / 2, &full[st]);
              load_w(dst + kASub + (N / 2) * kWRow, sg, sg.b_k0 + kc * 32, sg.b_n1, N / 2, &full[st]);
            } else {
              load_w(dst + kASub, sg, sg.b_k0 + kc * 32, sg.b_n0 + ncol0, N, &full[st]);
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

  // =============================== consumer warpgroup: wgmma mainloop + epilogue ===============================
  const int q = warp & 1;                 // rows 32 q .. 32 q + 31 of the tile in the epilogue
  const int hf = warp >> 1;               // 0 / 1: this warp takes 32-column chunks hf, hf + 2, ...
  const int row = q * 32 + lane;
  unsigned char* stg = stg_base + warp * 2 * kStg;
  const uint32_t ring_u32 = ptx::smem_u32(ring);
  uint32_t st = 0, ph = 0, nstore = 0;
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
    const int tt = tg * cm + rank;
    const int b = tt / tiles_per_b, t0 = (tt - b * tiles_per_b) * kTM;
    if (tt >= ntt) {   // past the last tile (partial last group): only keep the stages moving for the peers
      for (int kc = 0; kc < kchunks; kc++) {
        ptx::mbar_wait(&full[st], ph);
        release(st);
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      }
      continue;
    }
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[i] = 0.f;
    uint32_t prev = 0xFFFFFFFFu;
    if constexpr (!kBf16) {
      for (int kc = 0; kc < kchunks; kc++) {
        ptx::mbar_wait(&full[st], ph);
        ptx::wg_fence();
        const uint32_t a_addr = ring_u32 + st * stage_bytes, b_addr = a_addr + kASub;
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
      // A fragments (rows 16 warp + lane/4 (+ 8), k pairs 2 (lane % 4) (+ 8)) converted from the fp32 box into one of two
      // register sets: wgmma reads them asynchronously, so a set is refilled only after the chunk that used it is done
      const int fr = 16 * warp + (lane >> 2), fk = 2 * (lane & 3);
      uint32_t a0[2][4], a1[2][4];
      auto chunk = [&](uint32_t (&a)[2][4]) {
        ptx::mbar_wait(&full[st], ph);
        const unsigned char* as = ring + (size_t)st * stage_bytes;
#pragma unroll
        for (int k = 0; k < 2; k++)
#pragma unroll
          for (int h = 0; h < 4; h++) {
            const float2 v = *reinterpret_cast<const float2*>(as + ptx::sw128_off(fr + 8 * (h & 1), 16 * k + fk + 8 * (h >> 1)));
            a[k][h] = ptx::cvt_bf16x2(v.x, v.y);
          }
        ptx::wg_fence();
        const uint32_t b_addr = ring_u32 + st * stage_bytes + kASub;
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
    // accumulator -> shared memory (column-major), after every thread is done reading the previous tile's copy
    ptx::named_bar(1, kConsumers);
    {
      const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < N / 2; i++) accs[(8 * (i >> 2) + c0 + (i & 1)) * kAccLd + r0 + 8 * ((i >> 1) & 1)] = d[i];
    }
    ptx::named_bar(1, kConsumers);

    const int t = t0 + row;
    const bool row_ok = t < p.T;
    const size_t grow = (size_t)b * p.T + (row_ok ? t : 0);
    if constexpr (EPI == EPI_GATE_BWD_NOZ) {
      // ---- gate backward without the z output (the stack path): two passes of 16 gate channels; the two dpre boxes
      //      of this warp (d pre-sigmoid, d pre-tanh) are filled side by side and stored with one bulk group ----
      const int c0 = hf * 32;
      if (lane == 0) ptx::bulk_wait_read<0>();
      __syncwarp();
      const uint32_t sb0 = ptx::smem_u32(stg + lane * 128), sb1 = sb0 + kStg;
      const float4* bsv = reinterpret_cast<const float4*>(p.bias + c0);
      const float4* btv = reinterpret_cast<const float4*>(p.bias2 + c0);
      const float4* dzr = reinterpret_cast<const float4*>(p.gate_dz + grow * p.gate_ld_dz + p.gate_c0 + c0);
#pragma unroll
      for (int h2 = 0; h2 < 2; h2++) {
        const int cc = c0 + h2 * 16;
        float a[16], g[16], dzp[16];
        acc_ld16(accs, cc, row, a);
        acc_ld16(accs, 64 + cc, row, g);
        if (p.gate_mode == 3) acc_ld16(accs, 128 + cc, row, dzp);
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          const float4 d4 = row_ok ? __ldg(dzr + h2 * 4 + jj) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 bs = __ldg(bsv + h2 * 4 + jj), bt = __ldg(btv + h2 * 4 + jj);
          const float dzs[4] = {d4.x, d4.y, d4.z, d4.w};
          const float bsa[4] = {bs.x, bs.y, bs.z, bs.w}, bta[4] = {bt.x, bt.y, bt.z, bt.w};
          float da[4], dg[4];
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const int i = 4 * jj + k;
            float dz = dzs[k];
            if (p.gate_mode == 3) dz += dzp[i];
            const float sg = 0.5f * ptx::tanh_approx(0.5f * (a[i] + bsa[k])) + 0.5f;
            const float th = ptx::tanh_approx(g[i] + bta[k]);
            da[k] = dz * th * sg * (1.f - sg);      // d pre-sigmoid
            dg[k] = dz * sg * (1.f - th * th);      // d pre-tanh
          }
          const uint32_t off = (uint32_t)(((h2 * 4 + jj) ^ (lane & 7)) << 4);
          ptx::st_shared_v4(sb0 + off, da[0], da[1], da[2], da[3]);
          ptx::st_shared_v4(sb1 + off, dg[0], dg[1], dg[2], dg[3]);
        }
      }
      ptx::fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        ptx::tma_store_3d(&p.maps[9], stg, p.gate_c0 + c0, t0 + q * 32, b);
        ptx::tma_store_3d(&p.maps[9], stg + kStg, p.gate_R + p.gate_c0 + c0, t0 + q * 32, b);
        ptx::bulk_commit();
      }
      continue;
    }
    if constexpr (EPI == EPI_GATE) {
      // ---- gate epilogues: pair sigmoid column c with tanh column GC + c (GC = 64 or 128 gate channels per tile) ----
      const int GC = p.gate_gc;
      for (int c0 = hf * 32; c0 < GC; c0 += 64) {
        float a[32], g[32], dzv[32], dzp[32];
        acc_ld16(accs, c0, row, *reinterpret_cast<float(*)[16]>(a));
        acc_ld16(accs, c0 + 16, row, *reinterpret_cast<float(*)[16]>(a + 16));
        acc_ld16(accs, GC + c0, row, *reinterpret_cast<float(*)[16]>(g));
        acc_ld16(accs, GC + c0 + 16, row, *reinterpret_cast<float(*)[16]>(g + 16));
        if (p.gate_mode == 3) {
          acc_ld16(accs, 2 * GC + c0, row, *reinterpret_cast<float(*)[16]>(dzp));
          acc_ld16(accs, 2 * GC + c0 + 16, row, *reinterpret_cast<float(*)[16]>(dzp + 16));
        }
        if (p.gate_mode == 1) {
          // forward: z only
#pragma unroll
          for (int i = 0; i < 32; i++) {
            const float sg = 0.5f * ptx::tanh_approx(0.5f * (a[i] + __ldg(p.bias + c0 + i))) + 0.5f;
            dzv[i] = sg * ptx::tanh_approx(g[i] + __ldg(p.bias2 + c0 + i));
          }
          unsigned char* sb = stg + (nstore & 1) * kStg;
          if (lane == 0) ptx::bulk_wait_read<1>();
          __syncwarp();
          float4* dstrow = reinterpret_cast<float4*>(sb + lane * 128);
#pragma unroll
          for (int j = 0; j < 8; j++)
            dstrow[j ^ (lane & 7)] = make_float4(dzv[4 * j], dzv[4 * j + 1], dzv[4 * j + 2], dzv[4 * j + 3]);
          ptx::fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            ptx::tma_store_3d(&p.maps[8], sb, p.gate_c0 + c0, t0 + q * 32, b);
            ptx::bulk_commit();
          }
          nstore++;
          continue;
        }
        if (row_ok) {
          const float4* dr = reinterpret_cast<const float4*>(p.gate_dz + grow * p.gate_ld_dz + p.gate_c0 + c0);
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const float4 d4 = __ldg(dr + j);
            dzv[4 * j] = d4.x; dzv[4 * j + 1] = d4.y; dzv[4 * j + 2] = d4.z; dzv[4 * j + 3] = d4.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; i++) dzv[i] = 0.f;
        }
        if (p.gate_mode == 3) {
#pragma unroll
          for (int i = 0; i < 32; i++) dzv[i] += dzp[i];
        }
#pragma unroll
        for (int i = 0; i < 32; i++) {
          const float sg = 0.5f * ptx::tanh_approx(0.5f * (a[i] + __ldg(p.bias + c0 + i))) + 0.5f;
          const float th = ptx::tanh_approx(g[i] + __ldg(p.bias2 + c0 + i));
          const float dz = dzv[i];
          a[i] = dz * th * sg * (1.f - sg);      // d pre-sigmoid
          g[i] = dz * sg * (1.f - th * th);      // d pre-tanh
          dzv[i] = sg * th;                      // z
        }
#pragma unroll
        for (int which = 0; which < 3; which++) {
          if (which == 0 && p.gate_skip_z) continue;
          const float* src = which == 0 ? dzv : (which == 1 ? a : g);
          unsigned char* sb = stg + (nstore & 1) * kStg;
          if (lane == 0) ptx::bulk_wait_read<1>();
          __syncwarp();
          float4* dstrow = reinterpret_cast<float4*>(sb + lane * 128);
#pragma unroll
          for (int j = 0; j < 8; j++)
            dstrow[j ^ (lane & 7)] = make_float4(src[4 * j], src[4 * j + 1], src[4 * j + 2], src[4 * j + 3]);
          ptx::fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            if (which == 0) ptx::tma_store_3d(&p.maps[8], sb, p.gate_c0 + c0, t0 + q * 32, b);
            else ptx::tma_store_3d(&p.maps[9], sb, (which == 1 ? 0 : p.gate_R) + p.gate_c0 + c0, t0 + q * 32, b);
            ptx::bulk_commit();
          }
          nstore++;
        }
      }
      continue;
    }
    if constexpr (EPI == EPI_PLAIN) {
      for (int c0 = hf * 32; c0 < N; c0 += 64) {
        float v[32];
        acc_ld16(accs, c0, row, *reinterpret_cast<float(*)[16]>(v));
        acc_ld16(accs, c0 + 16, row, *reinterpret_cast<float(*)[16]>(v + 16));
        const bool second = p.out2_col0 > 0 && c0 >= p.out2_col0;
        if (p.bias && !second) {
#pragma unroll
          for (int i = 0; i < 32; i++) v[i] += __ldg(p.bias + ncol0 + c0 + i);
        }
        if (p.add && row_ok && !second) {
          const float4* ar = reinterpret_cast<const float4*>(p.add + grow * p.ldadd + ncol0 + c0);
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const float4 a = __ldg(ar + j);
            v[4 * j] += a.x; v[4 * j + 1] += a.y; v[4 * j + 2] += a.z; v[4 * j + 3] += a.w;
          }
        }
        if (p.relu_out && !second) {
#pragma unroll
          for (int i = 0; i < 32; i++) v[i] = fmaxf(v[i], 0.f);
        }
        if (p.mask && row_ok && !second) {
          const float4* mr = reinterpret_cast<const float4*>(p.mask + grow * p.ldmask + ncol0 + c0);
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const float4 m = __ldg(mr + j);
            v[4 * j] = m.x > 0.f ? v[4 * j] : 0.f; v[4 * j + 1] = m.y > 0.f ? v[4 * j + 1] : 0.f;
            v[4 * j + 2] = m.z > 0.f ? v[4 * j + 2] : 0.f; v[4 * j + 3] = m.w > 0.f ? v[4 * j + 3] : 0.f;
          }
        }
        unsigned char* sb = stg + (nstore & 1) * kStg;
        if (lane == 0) ptx::bulk_wait_read<1>();
        __syncwarp();
        float4* dstrow = reinterpret_cast<float4*>(sb + lane * 128);
#pragma unroll
        for (int j = 0; j < 8; j++)
          dstrow[j ^ (lane & 7)] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        ptx::fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          if (second) ptx::tma_reduce_add_3d(&p.maps[9], sb, c0 - p.out2_col0, t0 + q * 32, b);
          else if (p.accumulate) ptx::tma_reduce_add_3d(&p.maps[8], sb, ncol0 + c0, t0 + q * 32, b);
          else ptx::tma_store_3d(&p.maps[8], sb, ncol0 + c0, t0 + q * 32, b);
          ptx::bulk_commit();
        }
        nstore++;
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

// ngroups: cluster work items (p.cm time tiles x one column block); ctas: CTAs per SM the shared memory allows
template <int N, int EPI, typename W>
static cudaError_t launch_n(int ngroups, int ctas, size_t smem, cudaStream_t st, const Params& p) {
  cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(gemm_nt_tc_kernel<N, EPI, W>), smem);
  if (e != cudaSuccess) return e;
  int slots = device_sms() * ctas;
  if (p.cm > 1) {
    slots = max_active_clusters(gemm_nt_tc_kernel<N, EPI, W>, smem, p.cm);
    if (slots < 1) return cudaErrorInvalidConfiguration;
  }
  const int grid = (ngroups < slots ? ngroups : slots) * p.cm;
  return launch_pdl(gemm_nt_tc_kernel<N, EPI, W>, grid, kThreadsN, smem, st, p.cm, p);
}

template <int EPI, typename W>
static cudaError_t launch_epi(int N, int ngroups, int ctas, size_t smem, cudaStream_t st, const Params& p) {
  switch (N) {
    case 32: return launch_n<32, EPI, W>(ngroups, ctas, smem, st, p);
    case 64: return launch_n<64, EPI, W>(ngroups, ctas, smem, st, p);
    case 96: return launch_n<96, EPI, W>(ngroups, ctas, smem, st, p);
    case 128: return launch_n<128, EPI, W>(ngroups, ctas, smem, st, p);
    case 160: return launch_n<160, EPI, W>(ngroups, ctas, smem, st, p);
    case 192: return launch_n<192, EPI, W>(ngroups, ctas, smem, st, p);
    case 224: return launch_n<224, EPI, W>(ngroups, ctas, smem, st, p);
    default: return launch_n<256, EPI, W>(ngroups, ctas, smem, st, p);
  }
}

// CTAs per cluster for a launch whose weight boxes have box_rows rows (each half box, for the gate's two).
// The default is 1 for every launch.  Measured on an H100 80GB HBM3 (power limit not reported), bench.py's step
// (8 x 23 040, ms per step for the kind, CM = 1 / 2 / 4): skip GEMM 1.94 / 2.19 / 2.40, dZ_all 1.84 / 1.78 / 2.10, gate backward 4.62 / 4.77 /
// 5.24, dx 3.97 / 4.28 / 4.68; whole step 24.9 / 25.5 / 27.2 ms.  Halving the weight bytes pulled from L2 does not pay
// for the cluster-wide coupling of the ring while a tile's epilogue still runs after its mainloop in the same warpgroup.
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
  if (!map3(&p.maps[8], out, ld_out, T, B, 32)) { set_error("gemm_nt_tc: output map failed"); return WNB_ERR_CUDA; }
  p.maps[9] = p.maps[8];
  if (gate_dz) {   // R = 64 shorthand used by the fused-shape backward: whole gate in one launch
    const bool fused_dz = opts && opts->gate_fused_dz;
    if (N != (fused_dz ? 192 : 128) || !gate_dpre || !bias || !map3(&p.maps[9], gate_dpre, 128, T, B, 32)) {
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
    if (gate->mode == 2 && !map3(&p.maps[9], gate->dpre, 2 * gate->R, T, B, 32)) {
      set_error("gemm_nt_tc: dpre map failed");
      return WNB_ERR_CUDA;
    }
    for (int s = 0; s < nseg; s++) { p.seg[s].b_n0 = gate->c0; p.seg[s].b_n1 = gate->R + gate->c0; }
    p.bias = gate->bias_sig; p.bias2 = gate->bias_tanh; p.gate_dz = gate->dz;
    p.gate_mode = gate->mode; p.gate_c0 = gate->c0; p.gate_R = gate->R; p.gate_gc = GC;
  }
  if (out2) {
    if (gate_dz || out2_col0 <= 0 || out2_col0 % 32 != 0 || out2_col0 >= N || !map3(&p.maps[9], out2, ld_out2, T, B, 32)) {
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
  // shared memory: ring stages (A box + weight box) | accumulator copy | 4 warps x 2 staging boxes | barriers.  When three
  // stages fit in half of the SM, two CTAs share it and one's epilogue overlaps the other's mainloop.
  const int stage_bytes = kASub + N * (bf16 ? w_row_bytes<__nv_bfloat16>() : w_row_bytes<float>());
  const int fixed = acc_bytes(N) + 4 * 2 * kStg + 1024 + 256;
  const int sm_bytes = 227 * 1024, half = 113 * 1024;
  const int ctas = fixed + 3 * stage_bytes <= half ? 2 : 1;
  int nst = ((ctas == 2 ? half : sm_bytes) - fixed) / stage_bytes;
  if (nst > 6) nst = 6;
  if (nst < 2) { set_error("gemm_nt_tc: N too large"); return WNB_ERR_INVALID; }
  p.nstages = nst;
  const size_t smem = (size_t)fixed + (size_t)nst * stage_bytes;
  const int ngroups = cdiv(B * cdiv(T, kTM), p.cm) * p.nblk;
  cudaError_t le;
  if (bf16) {   // (the gate backward without z belongs to the tf32 stack only)
    if (epi == EPI_PLAIN) le = launch_epi<EPI_PLAIN, __nv_bfloat16>(N, ngroups, ctas, smem, st, p);
    else if (epi == EPI_GATE) le = launch_epi<EPI_GATE, __nv_bfloat16>(N, ngroups, ctas, smem, st, p);
    else { set_error("gemm_nt_tc: no bf16 variant of the gate backward without z"); return WNB_ERR_INVALID; }
  } else if (epi == EPI_PLAIN) le = launch_epi<EPI_PLAIN, float>(N, ngroups, ctas, smem, st, p);
  else if (epi == EPI_GATE) le = launch_epi<EPI_GATE, float>(N, ngroups, ctas, smem, st, p);
  else le = launch_epi<EPI_GATE_BWD_NOZ, float>(N, ngroups, ctas, smem, st, p);
  if (le != cudaSuccess) { set_error("gemm_nt_tc: launch failed: %s", cudaGetErrorString(le)); return WNB_ERR_CUDA; }
  WNB_CHECK_LAUNCH("gemm_nt_tc");
  return WNB_OK;
}

}  // namespace wnb
