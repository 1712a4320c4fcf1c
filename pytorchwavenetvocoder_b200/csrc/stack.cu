// stack.cu -- the whole residual stack of WaveNet.forward (reference wavenet.py:229-236 over :525-536) and its
// backward in "deferred skip" form, one C-ABI call each (WNB_MATH_TF32, n_resch = 64, kernel_size = 2, n_aux <= 32).
//
// The per-block formulation moves the (B,T,S) skip tensor through HBM in every block: a read-modify-write in the
// forward (skip += ...), and two reads in the backward (dz = dskip W2skip, dW2skip = dskip^T z) -- about 60 % of all
// bytes of a training step at 64 res / 512 skip channels.  Both directions are linear in the concatenated channel
// axis, so they are hoisted out of the block loop:
//
//   forward    z_l -> Z_all[:, :, l*R:(l+1)*R]     (resblock_z.cu writes the slice)
//              skip  = Z_all Wskip^T + bskip        one NT GEMM, K = L*R          (Wskip[s][l*R+c] = W2_l[R+s][c])
//   backward   dZ_all = dskip Wskip                  one NT GEMM, N = L*R in column blocks (A tile shared via L2)
//              per block: gate recompute + dz_l = dZ_all[l] + dout W2res_l + gate backward (one GEMM) ; dx, which is
//              the dout of the block below: dx_l and block l-1's gate backward run as one launch (stack_bwd_chain.cu)
//              dW1_l, dW2res_l of ALL blocks: one segmented weight-gradient launch each (dpre_l, dx_l are kept)
//              dWskip = dskip^T Z_all                one weight-gradient GEMM, column groups of Z_all across CTAs
//
// Z_all is written once and read twice per step (it replaces the z recompute output of the per-block backward).
#include <cuda_runtime.h>
#include <stdlib.h>

#include "../../include/wnb200.h"
#include "common.cuh"
#include "tc_host.h"

namespace wnb {

static int pick_block(int total, const int* cands, int n) {
  for (int i = 0; i < n; i++)
    if (total % cands[i] == 0) return cands[i];
  return 0;
}

// Consecutive kernels of the block chain walk the time tiles in opposite directions (forward: odd blocks backwards;
// backward: the chain launches alternately front to back and back to front), so each starts on the rows its producer
// wrote last -- still in the 50 MB L2 -- instead of on the ones written a tensor ago.  WNB_ALT_DIR=0: every kernel front
// to back.
static int alternate_dir() {
  static const int on = [] { const char* e = getenv("WNB_ALT_DIR"); return (e && e[0] == '0') ? 0 : 1; }();
  return on;
}

static bool stack_supported(int R, int S, int Ap, int ks, int L) {
  if (!resblock_fwd_z_supported(R, Ap, ks)) return false;
  if (L < 1 || L > 64 /* wnb_stack_bwd's segment shift table */) return false;
  if (S % 32 != 0 || S < 32 || (S > 256 && S != 512)) return false;
  return true;
}

}  // namespace wnb

using namespace wnb;

WNB_API int wnb_stack_supported(int R, int S, int Ap, int ks, int L, int math_mode) {
  return (math_mode == WNB_MATH_TF32 && stack_supported(R, S, Ap, ks, L)) ? 1 : 0;
}

WNB_API int wnb_resblock_fwd_z(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2res,
                               const float* b2res, float* xout, float* zall, int ldz, int zcol0, int B, int T, int R,
                               int Ap, int ks, int dilation, void* stream) {
  WNB_REQUIRE(B > 0 && T > 0 && dilation >= 1 && ldz >= R && zcol0 >= 0 && zcol0 + R <= ldz && ldz % 4 == 0,
              "resblock_fwd_z: bad shape");
  WNB_REQUIRE(xin && haux && w1 && b1 && zall && (!xout || (w2res && b2res)), "resblock_fwd_z: null pointer");
  if (!resblock_fwd_z_supported(R, Ap, ks)) {
    set_error("resblock_fwd_z: unsupported shape (R=%d Ap=%d ks=%d); use wnb_resblock_fwd", R, Ap, ks);
    return WNB_ERR_UNSUPPORTED;
  }
  return resblock_fwd_z(xin, haux, w1, b1, w2res, b2res, xout, zall, ldz, zcol0, B, T, dilation, (cudaStream_t)stream);
}

WNB_API int wnb_skip_gemm(const float* zall, const float* wskip, const float* bskip, float* skip, int B, int T, int K,
                          int S, int relu, void* stream) {
  WNB_REQUIRE(zall && wskip && skip && B > 0 && T > 0 && K % 32 == 0 && S % 32 == 0 && (S <= 256 || S == 512),
              "skip_gemm: bad arguments");
  const NtTcSeg seg[1] = {{zall, K, 0, K, wskip, S, K, 0, 0}};
  const int nblk = S > 256 ? S / 256 : 1;   // (a tile's accumulator is at most 256 columns)
  const NtTcOpts o{nblk};
  return gemm_nt_tc(seg, 1, S / nblk, skip, S, bskip, nullptr, 0, nullptr, 0, relu ? 1 : 0, 0, B, T, (cudaStream_t)stream,
                    nullptr, nullptr, nullptr, 0, 0, nullptr, &o);
}

WNB_API int wnb_stack_fwd(float* xs, int nxs, const float* haux, const float* w1, const float* b1, const float* w2res,
                          const float* b2res, const float* wskip, const float* bskip, float* zall, float* skip,
                          const int* dilations, int L, int B, int T, int R, int S, int Ap, int ks, int skip_relu,
                          void* stream) {
  WNB_REQUIRE(xs && haux && w1 && b1 && w2res && b2res && wskip && bskip && zall && skip && dilations,
              "stack_fwd: null pointer");
  WNB_REQUIRE(B > 0 && T > 0 && L >= 1 && nxs >= (L > 1 ? 2 : 1), "stack_fwd: bad shape");
  if (!stack_supported(R, S, Ap, ks, L)) {
    set_error("stack_fwd: unsupported shape (R=%d S=%d Ap=%d ks=%d)", R, S, Ap, ks);
    return WNB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t xsz = (size_t)B * T * R;
  const int K1 = ks * R + Ap, ldz = L * R;
  int rc;
  for (int l = 0; l < L; l++) {
    WNB_REQUIRE(dilations[l] >= 1, "stack_fwd: bad dilation");
    const float* xin = xs + (size_t)(l % nxs) * xsz;
    float* xout = (l + 1 < L) ? xs + (size_t)((l + 1) % nxs) * xsz : nullptr;
    ProfScope ps(WNB_PROF_FWD_BLOCK, st);
    if ((rc = resblock_fwd_z(xin, haux, w1 + (size_t)l * 2 * R * K1, b1 + (size_t)l * 2 * R, w2res + (size_t)l * R * R,
                             b2res + (size_t)l * R, xout, zall, ldz, l * R, B, T, dilations[l], st,
                             alternate_dir() ? (l & 1) : 0)) != WNB_OK)
      return rc;
  }
  ProfScope ps(WNB_PROF_SKIP_GEMM, st);
  return wnb_skip_gemm(zall, wskip, bskip, skip, B, T, ldz, S, skip_relu, stream);
}

// workspace: dZ_all (B,T,L*R) [+ one row of slack] | dpre of every block (L,B,T,2R) | dx of every block (L,B,T,R).
// dpre / dx of ALL blocks are kept so that the weight gradients dW1_l, dW2res_l of the whole stack are two launches at
// the end instead of 2L small ones inside the block loop (each of those spent a third of its time on launch, set-up
// and the atomic flush).
// On return wnb_stack_bwd leaves in it, in this order (floats):
//   dZ_all    B*T*L*R      dskip Wskip; columns l*R .. l*R+R-1 are block l's skip part of dz
//   slack     L*R          never written
//   dpre      L*B*T*2R     block l: [d pre-sigmoid | d pre-tanh] of its gate, the A operand of dW1_l
//   dx        L*B*T*R      block l >= 1: gradient of xs[l] (block l-1's dout, the A operand of dW2res_{l-1});
//                          slot 0 is never written (block 0's goes to dx0)
// tests/test_gpu_tc_stages.py reads these to check every stage from the kernels' own inputs.
WNB_API size_t wnb_stack_bwd_workspace(int L, int B, int T, int R, int S, int Ap, int ks) {
  (void)S; (void)Ap; (void)ks;
  const size_t bt = (size_t)B * T;
  return sizeof(float) * (bt * L * R + (size_t)L * R + (size_t)L * bt * 2 * R + (size_t)L * bt * R);
}

WNB_API int wnb_stack_bwd(const float* xs, const float* haux, const float* zall, const float* dskip, const float* w1,
                          const float* b1, const float* w1t, const float* wgate, const float* wskip_t, float* dx0,
                          float* dhaux, float* dw1, float* db1, float* dw2res, float* db2res, float* dwskip,
                          float* dbskip, void* workspace, const int* dilations, int L, int B, int T, int R, int S,
                          int Ap, int ks, void* stream) {
  WNB_REQUIRE(xs && haux && zall && dskip && w1 && b1 && w1t && wgate && wskip_t && dx0 && dw1 && db1 && dw2res &&
                  db2res && dwskip && dbskip && workspace && dilations,
              "stack_bwd: null pointer");
  WNB_REQUIRE(B > 0 && T > 0 && L >= 1, "stack_bwd: bad shape");
  if (!stack_supported(R, S, Ap, ks, L)) {
    set_error("stack_bwd: unsupported shape (R=%d S=%d Ap=%d ks=%d)", R, S, Ap, ks);
    return WNB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bt = (size_t)B * T, xsz = bt * R;
  const int K1 = ks * R + Ap, ldz = L * R;
  float* dzall = (float*)workspace;
  float* dpre_all = dzall + bt * ldz + ldz;                 // (L, B, T, 2R)
  float* dx_all = dpre_all + (size_t)L * bt * 2 * R;        // (L, B, T, R); slot 0 unused (block 0 writes dx0)
  WNB_REQUIRE(L <= 64, "stack_bwd: at most 64 blocks");
  int rc;

  {  // dZ_all = dskip Wskip   (wskip_t: rows n = l*R + c, K = S contiguous)
    static const int cands[] = {256, 192, 128, 64, 32};
    const int nb = pick_block(ldz, cands, 5);
    WNB_REQUIRE(nb > 0, "stack_bwd: L*R must be a multiple of 32");
    const NtTcSeg seg[1] = {{dskip, S, 0, S, wskip_t, ldz, S, 0, 0}};
    const NtTcOpts o{ldz / nb};
    ProfScope ps(WNB_PROF_DZALL_GEMM, st);
    if ((rc = gemm_nt_tc(seg, 1, nb, dzall, ldz, nullptr, nullptr, 0, nullptr, 0, 0, 0, B, T, st, nullptr, nullptr, nullptr,
                         0, 0, nullptr, &o)) != WNB_OK)
      return rc;
  }

  // The block chain in L + 1 launches: the gate backward of the last block alone, then one stack_bwd_chain launch per
  // block boundary l = L-1 .. 1 (dx_l, fed from shared memory straight into the gate backward of block l-1 as its dout),
  // then dx_0 alone.  Launch k walks the time tiles in direction k & 1.
  auto dpre_of = [&](int l) { return dpre_all + (size_t)l * bt * 2 * R; };
  auto dx_of = [&](int l) { return l == 0 ? dx0 : dx_all + (size_t)l * xsz; };
  auto wgate_of = [&](int l) { return wgate + (size_t)l * 3 * R * (K1 + R); };
  auto rev = [&](int launch) { return alternate_dir() ? (launch & 1) : 0; };
  {  // gate recompute (pre = W1 [x(t-d) | x(t) | aux]) and dz = dZ_all[L-1] -> dpre_{L-1}.  With a dout (the chain
     // kernel) the GEMM runs over the block matrix wgate_l = [[W1, 0], [0, W2res^T]] (3R x (K1+R)): accumulator
     // columns 2R..3R-1 are then the residual part of dz, dout W2res_l.
    const int l = L - 1, d = dilations[l];
    const float* xin = xs + (size_t)l * xsz;
    const float* wg = wgate_of(l);
    const NtTcSeg sg[3] = {{xin, R, -d, R, wg, 3 * R, K1 + R, 0, 0}, {xin, R, 0, R, wg, 3 * R, K1 + R, R, 0},
                           {haux, Ap, 0, Ap, wg, 3 * R, K1 + R, 2 * R, 0}};
    const NtTcOpts o{1, ldz, 1, 0, rev(0)};
    ProfScope ps(WNB_PROF_GATE_BWD, st);
    if ((rc = gemm_nt_tc(sg, 3, 2 * R, dx_of(l) /* z output suppressed */, R, b1 + (size_t)l * 2 * R, nullptr, 0,
                         nullptr, 0, 0, 0, B, T, st, dzall + (size_t)l * R, dpre_of(l), nullptr, 0, 0, nullptr, &o)) !=
        WNB_OK)
      return rc;
  }
  // dx_l = dx_{l+1} + dpre_l(t+d) W1_l[:, tap0] + dpre_l(t) W1_l[:, tap1]   and   dhaux += dpre_l(t) W1_l[:, aux]
  for (int l = L - 1; l >= 1; l--) {
    ProfScope ps(WNB_PROF_GATE_BWD, st);
    if ((rc = stack_bwd_chain(dpre_of(l), w1t + (size_t)l * K1 * 2 * R, l + 1 < L ? dx_of(l + 1) : nullptr, dx_of(l),
                              dhaux, xs + (size_t)(l - 1) * xsz, haux, wgate_of(l - 1), b1 + (size_t)(l - 1) * 2 * R,
                              dzall + (size_t)(l - 1) * R, ldz, dpre_of(l - 1), B, T, dilations[l], dilations[l - 1],
                              rev(L - l), st)) != WNB_OK)
      return rc;
  }
  {  // dx_0 (the same products and K order as the chain kernel's dX)
    const int d = dilations[0];
    const float* dpre = dpre_of(0);
    const float* dout = L > 1 ? dx_of(1) : nullptr;
    const NtTcOpts ox{1, 0, 0, 0, rev(L)};
    ProfScope ps(WNB_PROF_GATE_BWD, st);
    if (dhaux) {
      // (the shifted segment sees w1t as an R-row matrix: its rows R.. are TMA zero fill, only the unshifted tap feeds the
      //  aux columns)
      const NtTcSeg sx[2] = {{dpre, 2 * R, 0, 2 * R, w1t, K1, 2 * R, 0, R}, {dpre, 2 * R, d, 2 * R, w1t, R, 2 * R, 0, 0}};
      if ((rc = gemm_nt_tc(sx, 2, R + Ap, dx0, R, nullptr, nullptr, 0, dout, R, 0, 0, B, T, st, nullptr, nullptr, dhaux,
                           Ap, R, nullptr, &ox)) != WNB_OK)
        return rc;
    } else {
      const NtTcSeg sx[2] = {{dpre, 2 * R, d, 2 * R, w1t, K1, 2 * R, 0, 0}, {dpre, 2 * R, 0, 2 * R, w1t, K1, 2 * R, 0, R}};
      if ((rc = gemm_nt_tc(sx, 2, R, dx0, R, nullptr, nullptr, 0, dout, R, 0, 0, B, T, st, nullptr, nullptr, nullptr, 0, 0,
                           nullptr, &ox)) != WNB_OK)
        return rc;
    }
  }

  // The three weight gradients only read tensors that exist by now and do not depend on each other: ONE problem list,
  // one launch over every SM (wgrad_tc_multi), so the streaming-bound dW1 / dW2res stages run beside the
  // consumer-bound dWskip stages instead of after them.
  int seg_shift[64];
  for (int l = 0; l < L; l++) seg_shift[l] = -dilations[l];
  WgCall calls[3];
  int ncalls = 0;
  // every block's dW1 (128 x 160) += dpre_l^T [x_l(t-d_l) | x_l(t) | aux(t)], db1 = column sums of dpre_l: L segments
  WgBlock blk1;
  blk1.nops = 1;
  blk1.ops[0] = WgOperand{dpre_all, 2 * R, 0, 4, 0, WG_LAYERED, 0};
  blk1.c = dw1; blk1.m_valid = 128; blk1.db = db1;
  const WgOperand b1op[3] = {{xs, R, 0, 2, 0, WG_LAYERED | WG_SEG_SHIFT, 0}, {xs, R, 0, 2, 0, WG_LAYERED, 0},
                             {haux, Ap, 0, 1, 0, 0, 0}};
  calls[ncalls++] = WgCall{&blk1, 1, b1op, 3, K1, WgOpts{1, L, seg_shift, 2 * R * K1, 2 * R, 0}};
  // every block's dW2res (R x R) += dout_l^T z_l with dout_l = dx_{l+1} (an M = 64 problem: only its 2 sub-tiles are
  // loaded), db2res = column sums of dout_l; the last block has no residual output, hence L-1 segments
  WgBlock blk2;
  blk2.nops = 1;
  blk2.ops[0] = WgOperand{dx_all + xsz, R, 0, 4, 0, WG_LAYERED, 0};
  blk2.c = dw2res; blk2.m_valid = R; blk2.db = db2res;
  const WgOperand b2op[1] = {{zall, ldz, 0, R / 32, 0, 0, R}};
  if (L > 1) calls[ncalls++] = WgCall{&blk2, 1, b2op, 1, R, WgOpts{1, L - 1, seg_shift, R * R, R, 0}};
  // dWskip (S x L*R) += dskip^T Z_all, dbskip = column sums of dskip: every 128-row M-block of dskip, the L*R columns
  // of Z_all in column groups of up to 7 x 32
  const int groups = ldz / 32;
  const int nmb = (S + 127) / 128;
  int nB = 0;
  for (int c = 7; c >= 1 && !nB; c--)
    if (groups % c == 0 && groups / c <= 128) nB = c;
  WNB_REQUIRE(nB > 0, "stack_bwd: cannot split L*R into column groups");
  WNB_REQUIRE(nmb <= 5, "stack_bwd: at most 5 skip M-blocks");
  WgBlock blks[5];
  for (int i = 0; i < nmb; i++) {
    const int r = 128 * i;
    blks[i].nops = 1;
    blks[i].ops[0] = WgOperand{dskip, S, r, 4, 0, 0, 0};
    blks[i].c = dwskip + (size_t)r * ldz;
    blks[i].m_valid = (S - r) < 128 ? (S - r) : 128;
    blks[i].db = dbskip + r;
  }
  const WgOperand bsop[1] = {{zall, ldz, 0, nB, 0, 0, 0}};
  calls[ncalls++] = WgCall{blks, nmb, bsop, 1, ldz, WgOpts{groups / nB, 1, nullptr, 0, 0, 0}};
  ProfScope ps(WNB_PROF_WGRAD, st);
  return wgrad_tc_multi(calls, ncalls, B, T, st);
}
