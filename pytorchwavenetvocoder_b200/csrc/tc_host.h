// tc_host.h -- host-side entry points of the tensor-core (wgmma) kernels (internal; the C ABI is include/wnb200.h).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace wnb {

// ---- weight gradients (wgrad_tc.cu):  C_i[128 x N] += A_i^T B  over all (b, t) --------------------------------
// One operand = a channels-last tensor (B,T,C); `groups` 32-channel groups starting at channel c0, shifted in time.
enum { WG_LAYERED = 1,     // segment mode: the tensor is (nseg*B, T, C); segment i reads batches i*B ..
       WG_SEG_SHIFT = 2 }; // segment mode: time shift = WgOpts::seg_shift[i] instead of `shift`
struct WgOperand { const float* base; int C; int c0; int groups; int shift; int flags; int seg_cstride; };
// (seg_cstride: segment mode, channel offset added per segment -- a block's slice of a concatenated tensor)
// One M-block: 128 output rows = 4 groups taken from up to 2 operands (TMA zero fill past a tensor's channels).
struct WgBlock { WgOperand ops[2]; int nops; float* c; int m_valid; float* db; };
// n_split > 1: the B operand holds n_split consecutive column groups of 32*sum(groups_b) channels each, one problem
// per (M-block, column group); the problems of a call with several M-blocks or column groups share their operands
// through L2, so they are cut into equal time chunks that run side by side.  Bias gradients: column group 0 only.
// nseg > 1: nseg independent problems of identical structure (every residual block's dW1, say): operands pick their
// per-segment batch / shift / channel offsets with the WG_* flags, block i's C and db are at c + i*c_seg_stride,
// db + i*db_seg_stride.
// bf16: both operands are rounded to bf16 (nearest even) and multiplied by bf16 wgmma, fp32 accumulate.
struct WgOpts { int n_split; int nseg; const int* seg_shift; int c_seg_stride; int db_seg_stride; int bf16; };
// One call = the M-blocks of one B operand list.  wgrad_tc_multi runs the problems of all calls (same bf16 flag) as
// one launch of device_sms() CTAs plus one reduce; wgrad_tc_blocks / wgrad_tc are one-call lists.
struct WgCall { const WgBlock* blocks; int nblocks; const WgOperand* b_ops; int nb_ops; int ldc; WgOpts opts; };
int wgrad_tc_multi(const WgCall* calls, int ncalls, int B, int T, cudaStream_t st);
int wgrad_tc_blocks(const WgBlock* blocks, int nblocks, const WgOperand* b_ops, int nb_ops, int ldc, int B, int T,
                    cudaStream_t st, const WgOpts* opts = nullptr);
int wgrad_tc(const WgOperand* a_ops, int na_ops, const WgOperand* b_ops, int nb_ops, float* c, int ldc, int m_valid,
             float* db, int B, int T, cudaStream_t st);
// The static work split of one launch: problem i has stages[i] stages of cost[i] each, cut into nchunk[i] time chunks
// of ceil(stages / nchunk) stages (the unit one CTA sums from zero: it fixes the summation order); lock[i] != 0 marks
// problems that share operands through L2.  Writes CTA j's pieces (one chunk each) to pieces[cta_first[j] ..
// cta_first[j + 1]) (cta_first has sms + 1 entries; pieces may be null to count them) and returns the piece count, or
// -1 (bad input, or more than max_pieces).  A pure function of its arguments.
struct WgPiece { int prob, s0, s1; };
int wgrad_partition(const int* stages, const int* nchunk, const double* cost, const int* lock, int nprob, int sms,
                    int* cta_first, WgPiece* pieces, int max_pieces);

// ---- NT GEMM (gemm_nt_tc.cu):  out[b,t,n] = sum_seg sum_k A_seg[b,t+shift,k] W_seg[n0+n][k0+k]  (+ epilogues) ----
// One segment: activation tensor (B,T,CA) read at rows t+shift, channels [0,K); weight matrix w (rows x ldw,
// K-contiguous) rows [n0, n0+N), columns [k0, k0+K).  wb: null, or a bf16 copy of w (same layout): then both operands
// are rounded to bf16 (nearest even) and multiplied by bf16 wgmma; every segment of a call has one or none has.
struct NtTcSeg {
  const float* a; int CA; int shift; int K; const float* w; int w_rows; int w_cols; int k0; int n0;
  const __nv_bfloat16* wb;
};
// gate epilogue request: mode 1 = forward (z out), 2 = backward (dz in, z + dpre out); channels c0..c0+63 of R
struct NtTcGate { int mode; int c0; int R; const float* bias_sig; const float* bias_tanh; const float* dz; float* dpre; };
struct NtTcOpts {
  int n_blocks;      // > 1: N is one column block of n_blocks; block j uses weight rows n0 + j*N, output / bias / add /
                     //      mask columns j*N.. (tiles are ordered block-fastest, so the A tile is shared through L2)
  int gate_ld_dz;    // row pitch (floats) of the gate-backward dz input (0: gate_R)
  int gate_skip_z;   // gate-backward: do not write z
  int gate_fused_dz; // gate-backward shorthand with N == 192: accumulator columns 128..191 are added to dz
  int reverse;       // 1: time tiles are processed from the end of the tensor backwards (a kernel that consumes what the
                     //    previous launch wrote front to back finds the rows written last still in L2)
};
int gemm_nt_tc(const NtTcSeg* segs, int nseg, int N, float* out, int ld_out, const float* bias, const float* mask,
               int ldmask, const float* add, int ldadd, int relu_out, int accumulate, int B, int T, cudaStream_t st,
               const float* gate_dz = nullptr, float* gate_dpre = nullptr, float* out2 = nullptr, int ld_out2 = 0,
               int out2_col0 = 0, const NtTcGate* gate = nullptr, const NtTcOpts* opts = nullptr);

// ---- one block boundary of the stack backward (stack_bwd_chain.cu; R = 64, Ap = 32, ks = 2) ----------------------
// dx = dx_next + dpre(t) W1[:, tap1] + dpre(t+d) W1[:, tap0] (dx_next null: no residual), dhaux += dpre(t) W1[:, aux]
// (dhaux null: not computed), then the gate backward of the block below with dout = dx: gate recompute from
// [xprev(t-d_prev) | xprev(t) | haux] and dz = dz_prev (row pitch ldz) + dx W2res through wgate_prev, dpre_prev out.
// Bit-identical to gemm_nt_tc's dX launch followed by its N = 192 gate-backward launch.
int stack_bwd_chain(const float* dpre, const float* w1t, const float* dx_next, float* dx, float* dhaux, const float* xprev,
                    const float* haux, const float* wgate_prev, const float* b1_prev, const float* dz_prev, int ldz,
                    float* dpre_prev, int B, int T, int d, int d_prev, int reverse, cudaStream_t st);

// ---- fused residual block, deferred-skip form (resblock_z.cu) --------------------------------------------------
bool resblock_fwd_z_supported(int R, int Ap, int ks);
int resblock_fwd_z(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2res,
                   const float* b2res, float* xout, float* zall, int ldz, int zcol0, int B, int T, int d,
                   cudaStream_t st, int reverse = 0);   // reverse: time tiles from the end of the tensor backwards

// ---- fused residual block, per-block form with skip accumulation (resblock_z.cu) ----------------------------------
bool resblock_fwd_skip_supported(int R, int S, int Ap, int ks);
int resblock_fwd_skip(const float* xin, const float* haux, const float* w1, const float* b1, const float* w2,
                      const float* b2, float* xout, float* skip, int B, int T, int S, int d, int skip_init,
                      cudaStream_t st);

}  // namespace wnb
