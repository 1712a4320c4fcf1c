// stack_bwd_chain.cu -- one launch per block boundary of the stack backward (csrc/stack.cu, R = 64, ks = 2, Ap = 32,
// tf32): block l's data gradient dX and the gate backward of block l-1, whose dout is that dx.
//
//   dx_l(t)   = dx_{l+1}(t) + dpre_l(t) W1_l[:, tap1] + dpre_l(t + d_l) W1_l[:, tap0]     (-> dx_all[l] or dx0)
//   dhaux(t) += dpre_l(t) W1_l[:, aux]                                                     (TMA reduce-add)
//   gate backward of block l-1 at row t: recompute pre = W1_{l-1} [x(t-d) | x(t) | aux(t)], dz = dZ_all[l-1](t) +
//   dx_l(t) W2res_{l-1}, dpre_{l-1} out -- one GEMM over wgate_{l-1} (192 x 224), as gemm_nt_tc's N = 192 gate backward.
//
// dx_l(t) reads only dpre_l, which the previous launch wrote completely; the gate backward at row t needs dx_l at row t
// only.  So a consumer warpgroup computes a 64-row tile of dx_l, stores it, and writes the same fp32 values into a
// swizzled K-major [64 x 64] shared-memory tile that is the A operand of the gate GEMM's dout segment: dout is never read
// back from HBM.  Every product keeps gemm_nt_tc's instruction shape, operands, K order and epilogue arithmetic (dX: the
// plain epilogue with residual and split dhaux output; gate: the no-z gate backward), so the results are bit-identical
// to the two launches it replaces.
//
// Structure as gemm_nt_tc (DESIGN 3.1): one producer warpgroup (one TMA thread, setmaxnreg 40) and two consumer
// warpgroups (232) on pairs of consecutive 64-row time tiles; per stage of the ring the producer loads both tiles'
// [64 x 32] activation boxes and ONE weight box that both warpgroups multiply.  A tile pair takes 15 stages: 8 of the dX
// GEMM (dpre_l, w1t_l boxes of NX rows), 5 of the gate GEMM's x(t-d), x(t), aux segments and 2 of its dout segment,
// whose A operand is the dx_l tile in shared memory: their activation slots carry the two [64 x 32] boxes of the
// dZ_all[l-1] slice instead, which each thread copies into registers for the gate epilogue.  The residual dx_{l+1} tile
// is staged by TMA when the tile starts and then becomes the dout tile (each thread overwrites the residual values it
// has just added).  No per-tile dz buffer is needed, which leaves room for a fourth ring stage.  Epilogues run from
// registers through per-warp staging boxes and TMA stores.
#include <cuda.h>
#include <string.h>

#include "common.cuh"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace wnb {
namespace chain {

constexpr int kR = 64, kAp = 32, kK1 = 2 * kR + kAp;   // K1 = 160: [x(t-d) | x(t) | aux] columns of W1
constexpr int kTM = 64;                                 // time rows per tile (wgmma M)
constexpr int kASub = kTM * 32 * 4;                     // 8 KB: one tile's activation box of a stage
constexpr int kNG = 3 * kR;                             // 192: gate GEMM columns [sigmoid | tanh | dz partial]
constexpr int kStage = 2 * kASub + kNG * 128;           // 40 KB: [A box tile 0 | A box tile 1 | weight box]
constexpr int kStgRows = 16;
constexpr int kStg = kStgRows * 32 * 4;                 // 2 KB staging box: one warp's 16 rows x 32 columns
constexpr int kStgBytes = 8 * 2 * kStg;                 // 8 consumer warps x 2 staging boxes
constexpr int kEopBox = kTM * 32 * 4;                   // 8 KB: [64 x 32] box
constexpr int kEopWG = 2 * kEopBox;                     // per warpgroup: residual / dout tile (2 boxes)
constexpr int kWG = 128;
constexpr int kConsumers = 2 * kWG;
constexpr int kThreads = kConsumers + kWG;
constexpr int kDxChunks = 8, kGateTmaChunks = 5, kChunks = kDxChunks + kGateTmaChunks + 2;

struct alignas(64) Params {
  // [0] dpre_l  [1] x_{l-1}  [2] aux  [3] w1t_l (K1 rows)  [4] w1t_l as an R-row matrix  [5] wgate_{l-1}
  // [6] dx_l out  [7] dhaux (reduce-add)  [8] dpre_{l-1} out  [9] dx_{l+1} (residual)  [10] dZ_all[l-1] slice
  CUtensorMap maps[11];
  const float* bias;    // b1_{l-1}: sigmoid bias, tanh bias at + 64
  int B, T, nstages, d_l, d_prev, has_res, rev;
};

// the operands of chunk c (0 .. kChunks-1) of a tile: the box loaded into the stage's activation slot (map, column, time
// shift; in the two dout chunks a dz box, not an MMA operand) and the weight box (map, k, first row)
template <bool AUX>
__device__ __forceinline__ void chunk_src(const Params& p, int c, int& amap, int& acol, int& shift, int& wmap, int& wk,
                                          int& wn) {
  if (c < kDxChunks) {
    // with dhaux: dpre(t) against w1t rows R .. 2R+Ap-1 ([tap1 | aux]), then dpre(t+d) against rows 0 .. R-1 (the R-row
    // map zero-fills the aux rows); without: dpre(t+d) against rows 0 .. R-1, then dpre(t) against rows R .. 2R-1
    const bool first = c < 4, shifted = AUX ? !first : first;
    amap = 0; acol = 32 * (c & 3); shift = shifted ? p.d_l : 0;
    wmap = (AUX && !first) ? 4 : 3; wk = 32 * (c & 3); wn = shifted ? 0 : kR;
    return;
  }
  const int g = c - kDxChunks;   // gate: x(t-d) (2 chunks), x(t) (2), aux (1), dout (2); wgate columns in that order
  wmap = 5; wk = 32 * g; wn = 0;
  if (g < 4) { amap = 1; acol = 32 * (g & 1); shift = g < 2 ? -p.d_prev : 0; }
  else if (g == 4) { amap = 2; acol = 0; shift = 0; }
  else { amap = 10; acol = 32 * (g - 5); shift = 0; }
}

template <bool AUX>
__global__ void __launch_bounds__(kThreads, 1) stack_bwd_chain_kernel(const __grid_constant__ Params p) {
  constexpr int NX = AUX ? kR + kAp : kR;   // dX GEMM columns: [dx | dhaux part]
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* ring = smem;
  unsigned char* stg_base = ring + (size_t)p.nstages * kStage;
  unsigned char* eop_base = stg_base + kStgBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(eop_base + 2 * kEopWG);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.nstages;
  uint64_t* res_full = bars + 2 * p.nstages;   // [2]: per consumer warpgroup
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_b = (p.T + kTM - 1) / kTM;
  const int ntt = p.B * tiles_per_b;
  const int npairs = (ntt + 1) / 2;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; i++) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kConsumers / 32);
    }
    for (int i = 0; i < 2; i++) ptx::mbar_init(&res_full[i], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch: dpre_l is the previous launch's output
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();

  if (warp >= kConsumers / 32) {
    // =============================== TMA producer warpgroup ===============================
    ptx::setmaxnreg_dec<40>();
    if (warp == kConsumers / 32 && ptx::elect_one()) {
      for (int i = 0; i < 11; i++) ptx::prefetch_tmap(&p.maps[i]);
      uint32_t st = 0, ph = 0;
      for (int grp = blockIdx.x; grp < npairs; grp += gridDim.x) {
        const int tt0 = 2 * (p.rev ? npairs - 1 - grp : grp);
        const int ntiles = tt0 + 1 < ntt ? 2 : 1;
        int tb[2], tt[2];
#pragma unroll
        for (int h = 0; h < 2; h++) { tb[h] = (tt0 + h) / tiles_per_b; tt[h] = (tt0 + h - tb[h] * tiles_per_b) * kTM; }
        for (int c = 0; c < kChunks; c++) {
          int amap, acol, shift, wmap, wk, wn;
          chunk_src<AUX>(p, c, amap, acol, shift, wmap, wk, wn);
          const int wbytes = (c < kDxChunks ? NX : kNG) * 128;
          ptx::mbar_wait<ptx::kStoreFault>(&empty[st], ph ^ 1);
          ptx::mbar_arrive_expect_tx(&full[st], wbytes + ntiles * kASub);
          unsigned char* dst = ring + (size_t)st * kStage;
          for (int h = 0; h < ntiles; h++) ptx::tma_load_3d(dst + h * kASub, &p.maps[amap], &full[st], acol, tt[h] + shift, tb[h]);
          ptx::tma_load_2d(dst + 2 * kASub, &p.maps[wmap], &full[st], wk, wn);
          if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  ptx::setmaxnreg_inc<232>();
  const int wg = warp >> 2, wq = warp & 3;
  const int rq = lane >> 2, cq = 2 * (lane & 3);
  const int r16 = 16 * wq;
  unsigned char* stg = stg_base + warp * 2 * kStg;
  unsigned char* dout_tile = eop_base + wg * kEopWG;   // residual dx_{l+1}, then dx_l: the gate GEMM's dout operand
  const uint32_t ring_u32 = ptx::smem_u32(ring), dout_u32 = ptx::smem_u32(dout_tile);
  uint32_t st = 0, ph = 0, nstore = 0, rph = 0;
  auto release = [&](uint32_t s) {
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  };
  for (int grp = blockIdx.x; grp < npairs; grp += gridDim.x) {
    const int tt = 2 * (p.rev ? npairs - 1 - grp : grp) + wg;
    const int b = tt / tiles_per_b, t0 = (tt - b * tiles_per_b) * kTM;
    if (tt >= ntt) {   // the second tile of a partial last pair: only keep the stages moving
      for (int c = 0; c < kChunks; c++) {
        ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
        release(st);
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      }
      continue;
    }
    // this tile's residual, once every warp of the warpgroup is done with the previous tile's dout tile
    ptx::named_bar(1 + wg, kWG);
    if (p.has_res && wq == 0 && lane == 0) {
      ptx::mbar_arrive_expect_tx(&res_full[wg], 2 * kEopBox);
      for (int k = 0; k < 2; k++) ptx::tma_load_3d(dout_tile + k * kEopBox, &p.maps[9], &res_full[wg], 32 * k, t0, b);
    }
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

    // ---- dX GEMM: chunks 0 .. 7 ----
    {
      float d[NX / 2];
#pragma unroll
      for (int i = 0; i < NX / 2; i++) d[i] = 0.f;
      uint32_t prev = 0xFFFFFFFFu;
      for (int c = 0; c < kDxChunks; c++) {
        ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
        ptx::wg_fence();
        const uint32_t a_addr = ring_u32 + st * kStage + wg * kASub, b_addr = ring_u32 + st * kStage + 2 * kASub;
#pragma unroll
        for (int k = 0; k < 4; k++)
          ptx::wgmma_ss<NX>(d, ptx::gmma_desc_k_sw128(a_addr + 32 * k), ptx::gmma_desc_k_sw128(b_addr + 32 * k), 1);
        ptx::wg_commit();
        ptx::wg_wait<1>();
        if (prev != 0xFFFFFFFFu) release(prev);
        prev = st;
        if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
      }
      ptx::wg_wait<0>();
      ptx::wg_touch(d);
      release(prev);
      if (p.has_res) {
        ptx::mbar_wait<ptx::kStoreFault>(&res_full[wg], rph);
        rph ^= 1;
      }
      // value v[4 jj + 2 h + e] of 32-column chunk cb: row r16 + rq + 8 h, column 32 cb + 8 jj + cq + e
#pragma unroll
      for (int cb = 0; cb < NX / 32; cb++) {
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; i++) v[i] = d[16 * cb + i];
        if (cb < kR / 32) {   // dx = acc + dx_{l+1}: stored, and kept as the gate GEMM's dout tile
#pragma unroll
          for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
              float2* e = reinterpret_cast<float2*>(dout_tile + cb * kEopBox + ptx::sw128_off(r16 + rq + 8 * h, 8 * jj + cq));
              if (p.has_res) {
                const float2 a = *e;
                v[4 * jj + 2 * h] += a.x; v[4 * jj + 2 * h + 1] += a.y;
              }
              *e = make_float2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
            }
          store16(v, &p.maps[6], 32 * cb, false);
        } else {
          store16(v, &p.maps[7], 32 * cb - kR, true);
        }
      }
    }
    // the dout tile written by every warp of the warpgroup -> visible to its wgmma (async proxy)
    ptx::fence_proxy_async();
    ptx::named_bar(1 + wg, kWG);

    // ---- gate GEMM of block l-1: chunks 8 .. 14 (the last two with A = the dout tile, and this tile's dz boxes in the
    //      activation slot: dzr[cb][jj][h] = dz at row r16 + rq + 8 h, columns 32 cb + 8 jj + cq, + 1) ----
    float2 dzr[2][4][2];
    float d[kNG / 2];
#pragma unroll
    for (int i = 0; i < kNG / 2; i++) d[i] = 0.f;
    uint32_t prev = 0xFFFFFFFFu;
    for (int g = 0; g < kChunks - kDxChunks; g++) {
      ptx::mbar_wait<ptx::kStoreFault>(&full[st], ph);
      if (g >= kGateTmaChunks) {
        const unsigned char* dzb = ring + (size_t)st * kStage + wg * kASub;
#pragma unroll
        for (int jj = 0; jj < 4; jj++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const float2 v = *reinterpret_cast<const float2*>(dzb + ptx::sw128_off(r16 + rq + 8 * h, 8 * jj + cq));
            if (g == kGateTmaChunks) dzr[0][jj][h] = v;
            else dzr[1][jj][h] = v;
          }
      }
      ptx::wg_fence();
      const uint32_t a_addr = g < kGateTmaChunks ? ring_u32 + st * kStage + wg * kASub
                                                 : dout_u32 + (g - kGateTmaChunks) * kEopBox;
      const uint32_t b_addr = ring_u32 + st * kStage + 2 * kASub;
#pragma unroll
      for (int k = 0; k < 4; k++)
        ptx::wgmma_ss<kNG>(d, ptx::gmma_desc_k_sw128(a_addr + 32 * k), ptx::gmma_desc_k_sw128(b_addr + 32 * k), 1);
      ptx::wg_commit();
      ptx::wg_wait<1>();
      if (prev != 0xFFFFFFFFu) release(prev);
      prev = st;
      if (++st == (uint32_t)p.nstages) { st = 0; ph ^= 1; }
    }
    ptx::wg_wait<0>();
    ptx::wg_touch(d);
    release(prev);
    // gate backward epilogue: sigmoid column c pairs with tanh column 64 + c (d[i + 32]) and the dz partial at 128 + c
    // (d[i + 64]); dpre_{l-1} = [d pre-sigmoid | d pre-tanh], z not written
#pragma unroll
    for (int cb = 0; cb < 2; cb++) {
      float a[16], g[16];
#pragma unroll
      for (int jj = 0; jj < 4; jj++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int c = 32 * cb + 8 * jj + cq, v = 4 * jj + 2 * h, i = 4 * (4 * cb + jj) + 2 * h;
          const float2 dz2 = dzr[cb][jj][h];
          const float dzs[2] = {dz2.x, dz2.y};
          const float bsa[2] = {__ldg(p.bias + c), __ldg(p.bias + c + 1)};
          const float bta[2] = {__ldg(p.bias + kR + c), __ldg(p.bias + kR + c + 1)};
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const float sg = 0.5f * ptx::tanh_approx(0.5f * (d[i + e] + bsa[e])) + 0.5f;
            const float th = ptx::tanh_approx(d[i + e + 32] + bta[e]);
            float dz = dzs[e];
            dz += d[i + e + 64];
            a[v + e] = dz * th * sg * (1.f - sg);      // d pre-sigmoid
            g[v + e] = dz * sg * (1.f - th * th);      // d pre-tanh
          }
        }
      store16(a, &p.maps[8], 32 * cb, false);
      store16(g, &p.maps[8], kR + 32 * cb, false);
    }
  }
  if (lane == 0) ptx::bulk_wait<0>();
  __syncwarp();
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
// (B,T,C) channels-last tensor with row pitch ld, [box_rows x 32] boxes; [K x Nrows] row-major weight matrix, [box_rows x
// 32] boxes.  128B swizzle, zero fill outside the tensor: the layouts of gemm_nt_tc.
static bool map3(CUtensorMap* m, const float* base, int ld, int T, int B, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[3] = {(cuuint64_t)ld, (cuuint64_t)T, (cuuint64_t)B};
  cuuint64_t gstr[2] = {(cuuint64_t)ld * 4, (cuuint64_t)ld * 4 * (cuuint64_t)T};
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

template <bool AUX>
static cudaError_t launch(int npairs, size_t smem, cudaStream_t st, const Params& p) {
  cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(stack_bwd_chain_kernel<AUX>), smem);
  if (e != cudaSuccess) return e;
  const int grid = npairs < device_sms() ? npairs : device_sms();
  return launch_pdl(stack_bwd_chain_kernel<AUX>, grid, kThreads, smem, st, 1, p);
}

}  // namespace chain

int stack_bwd_chain(const float* dpre, const float* w1t, const float* dx_next, float* dx, float* dhaux, const float* xprev,
                    const float* haux, const float* wgate_prev, const float* b1_prev, const float* dz_prev, int ldz,
                    float* dpre_prev, int B, int T, int d, int d_prev, int reverse, cudaStream_t st) {
  using namespace chain;
  // TMA needs 16-byte aligned bases; the bias is read in float2 pairs
  const auto al16 = [](const void* ptr) { return !(reinterpret_cast<uintptr_t>(ptr) & 15); };
  if (!dpre || !w1t || !dx || !xprev || !haux || !wgate_prev || !b1_prev || !dz_prev || !dpre_prev || B < 1 || T < 1 ||
      d < 1 || d_prev < 1 || ldz % 4 != 0 || ldz < kR || !al16(dz_prev) || (dx_next && !al16(dx_next)) ||
      (dhaux && !al16(dhaux)) || (reinterpret_cast<uintptr_t>(b1_prev) & 7)) {
    set_error("stack_bwd_chain: bad arguments");
    return WNB_ERR_INVALID;
  }
  Params p;
  memset(&p, 0, sizeof(p));
  const int NX = dhaux ? kR + kAp : kR;
  bool ok = map3(&p.maps[0], dpre, 2 * kR, T, B, kTM) && map3(&p.maps[1], xprev, kR, T, B, kTM) &&
            map3(&p.maps[2], haux, kAp, T, B, kTM) && map2(&p.maps[3], w1t, 2 * kR, kK1, NX) &&
            map2(&p.maps[4], w1t, 2 * kR, kR, NX) && map2(&p.maps[5], wgate_prev, kK1 + kR, kNG, kNG) &&
            map3(&p.maps[6], dx, kR, T, B, kStgRows) && map3(&p.maps[8], dpre_prev, 2 * kR, T, B, kStgRows) &&
            map3(&p.maps[10], dz_prev, ldz, T, B, kTM);
  ok = ok && (dhaux ? map3(&p.maps[7], dhaux, kAp, T, B, kStgRows) : (p.maps[7] = p.maps[6], true));
  ok = ok && (dx_next ? map3(&p.maps[9], dx_next, kR, T, B, kTM) : (p.maps[9] = p.maps[6], true));
  if (!ok) {
    set_error("stack_bwd_chain: tensor map creation failed");
    return WNB_ERR_CUDA;
  }
  p.bias = b1_prev;
  p.B = B; p.T = T; p.d_l = d; p.d_prev = d_prev; p.has_res = dx_next ? 1 : 0; p.rev = reverse ? 1 : 0;
  // shared memory: ring stages | 8 warps x 2 staging boxes | 2 warpgroups x dout tile | barriers
  const int fixed = kStgBytes + 2 * kEopWG + 1024 + 256;
  int nst = (227 * 1024 - fixed) / kStage;
  if (nst > 6) nst = 6;
  p.nstages = nst;
  const size_t smem = (size_t)fixed + (size_t)nst * kStage;
  const int npairs = cdiv(B * cdiv(T, kTM), 2);
  const cudaError_t le = dhaux ? launch<true>(npairs, smem, st, p) : launch<false>(npairs, smem, st, p);
  if (le != cudaSuccess) { set_error("stack_bwd_chain: launch failed: %s", cudaGetErrorString(le)); return WNB_ERR_CUDA; }
  WNB_CHECK_LAUNCH("stack_bwd_chain");
  return WNB_OK;
}

}  // namespace wnb
