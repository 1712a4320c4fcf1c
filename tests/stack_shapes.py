# -*- coding: utf-8 -*-
"""The shape table of tests/test_gpu_stack_shapes.py and tests/test_stack_shapes_host.py: the tf32 deferred-skip stack
(``wnb_stack_fwd`` / ``wnb_stack_bwd``: csrc/stack.cu, csrc/resblock_z.cu, csrc/stack_bwd_chain.cu) and the fused
R = 64 per-block path (``resblock_fwd_skip`` with the R = 64 gate-GEMM backward of ``wnb_resblock_bwd``) across their
whole coverage.

``stack_supported`` takes R 64, ks 2, Ap 32 with L in 1..64 and S in {32, 64, ..., 256, 512}; a model whose shape it
does not take but whose S is a multiple of 64 (S in {320, 384, 448, 576, ...}, or more than 64 blocks) trains on the
fused per-block path.  Each launch of either path is a template instantiation or a split of the work that depends on
the shape (tests/test_stack_shapes_host.py restates the dispatch and names them); the rows together reach every one
that the coverage grid reaches, with the aux gradient on and off.

Stack rows: ``L, S, B, T, dilations``, ``relu`` (the skip GEMM's ReLU epilogue), ``aux`` (dhaux is computed: off for a
model without an up-sampling layer), and ``reaches``.  Every skip width meets L in {1, 2, 3, 5, 7} (dWskip nB 2, 4, 6,
5, 7 -- every nB of the coverage); L = 4 adds the one-block dZ_all of 256 columns, L = 59 at S = 512 a weight-gradient
list of 353 problems (three launches of ``kMaxProb`` = 160) and L = 64 at S = 512 one of 255 (two); the six cases of
test_gpu_tc_stages.test_stack_stages are kept as they were (case d's T is derived from the SM count there).  ``aux``
alternates so that both chain kernel templates meet the first launch (no residual) and the later ones (a residual, both
tile directions), and dx_0 meets L = 1, even L and odd L both ways.  Time profiles cycle through T = 1, T < 64 with L >=
2 (one tile per utterance in every chain launch), T one under and one over a multiple of 64, odd 64-row tile counts over
B = 1 (a half-empty last pair) and B = 3 (pairs spanning utterances); dilations cycle so that some d_l >= T and
neighbouring d_l, d_{l-1} lie 256 and more apart.

Fused rows (R 64, ks 2, Ap 32): ``S, d, B, T``, ``last`` (dout is NULL: no residual chunk, dW2 from row R), ``init``
(skip is stored rather than accumulated), ``aux`` (dhaux is computed).  Between them they reach every (M-blocks,
[dout | dskip] block, M = 64 form) of the dW2 launches -- a launch every 5 M-blocks and after the last, R + S > 640
with and without dout, R + S - row_first a multiple of 128 and not -- both dX forms with and without dout, and W2
chunk counts (S/64, + 1 with a residual) that are and are not a multiple of the forward's 2-slot ring, with ``init``
both ways."""


def _row(L, S, B, T, dilations, relu, aux, reaches):
    return dict(L=L, S=S, B=B, T=T, dilations=list(dilations), relu=relu, aux=aux, reaches=reaches)


# the cases of test_gpu_tc_stages.test_stack_stages (run there with relu 0 and 1)
STAGE_CASES = ("a", "b", "c", "d", "e", "f")

STACK_ROWS = {
    # ---- the six stage cases ----
    "case_a": _row(1, 32, 1, 1, [1], relu=0, aux=True,
                   reaches="a one-row tile, d >= T, no dW2res launch, ldz = 64"),
    "case_b": _row(3, 96, 2, 95, [1, 64, 200], relu=0, aux=True,
                   reaches="partial 64- and 32-row tiles, d > T, dWskip m_valid = 96"),
    "case_c": _row(5, 512, 3, 1040, [1, 2, 4, 8, 16], relu=0, aux=True,
                   reaches="dZ_all in five 64-column blocks, skip GEMM in 2 blocks, 4 dWskip M-blocks"),
    "case_d": _row(22, 256, 1, None, [2 ** (i % 10) for i in range(22)], relu=0, aux=True,
                   reaches="weight-gradient CTAs with an empty time range in dW1, dW2res and dWskip"),
    "case_e": _row(30, 512, 2, 8300, [2 ** i for i in range(10)] * 3, relu=0, aux=True,
                   reaches="several tiles per CTA in every kernel, reversed tile order on odd blocks"),
    "case_f": _row(64, 128, 1, 200, [(37 * i) % 300 + 1 for i in range(64)], relu=0, aux=True,
                   reaches="64 segments (the limit), dZ_all in 16 blocks, dWskip n_split = 32"),
    # ---- every skip width x L in {1, 2, 3, 5, 7} ----
    'l1_s32': _row(1, 32, 1, 1, [1], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 32 rows, nB 2 x 1, M64; dZ_all 64 x 1; no chain; dx_0 no dhaux, L 1'),
    'l2_s32_aux': _row(2, 32, 2, 40, [300, 2], relu=0, aux=True,
        reaches='dWskip 1 M-block, last 32 rows, nB 4 x 1; dZ_all 128 x 1; chain with dhaux; dx_0 with dhaux, even L'),
    'l3_s32': _row(3, 32, 2, 127, [2, 64, 512], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 32 rows, nB 6 x 1; dZ_all 192 x 1; chain no dhaux; dx_0 no dhaux, odd L'),
    'l5_s32_aux': _row(5, 32, 1, 129, [64, 512, 3, 130, 1], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 32 rows, nB 5 x 2; dZ_all 64 x 5; chain with dhaux; dx_0 with dhaux, odd L'),
    'l7_s32': _row(7, 32, 3, 63, [512, 3, 130, 1, 300, 2, 64], relu=1, aux=False,
        reaches='dWskip 1 M-block, last 32 rows, nB 7 x 2; dZ_all 64 x 7; chain no dhaux; dx_0 no dhaux, odd L'),
    'l1_s64_aux': _row(1, 64, 3, 129, [3], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 64 rows, nB 2 x 1, M64; dZ_all 64 x 1; no chain; dx_0 with dhaux, L 1'),
    'l2_s64': _row(2, 64, 1, 1, [130, 1], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 64 rows, nB 4 x 1; dZ_all 128 x 1; chain no dhaux; dx_0 no dhaux, even L'),
    'l3_s64_aux': _row(3, 64, 2, 40, [1, 300, 2], relu=0, aux=True,
        reaches='dWskip 1 M-block, last 64 rows, nB 6 x 1; dZ_all 192 x 1; chain with dhaux; dx_0 with dhaux, odd L'),
    'l5_s64': _row(5, 64, 2, 127, [300, 2, 64, 512, 3], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 64 rows, nB 5 x 2; dZ_all 64 x 5; chain no dhaux; dx_0 no dhaux, odd L'),
    'l7_s64_aux': _row(7, 64, 1, 129, [2, 64, 512, 3, 130, 1, 300], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 64 rows, nB 7 x 2; dZ_all 64 x 7; chain with dhaux; dx_0 with dhaux, odd L'),
    'l1_s96': _row(1, 96, 3, 63, [64], relu=1, aux=False,
        reaches='dWskip 1 M-block, last 96 rows, nB 2 x 1; dZ_all 64 x 1; no chain; dx_0 no dhaux, L 1'),
    'l2_s96_aux': _row(2, 96, 3, 129, [512, 3], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 96 rows, nB 4 x 1; dZ_all 128 x 1; chain with dhaux; dx_0 with dhaux, even L'),
    'l3_s96': _row(3, 96, 1, 1, [3, 130, 1], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 96 rows, nB 6 x 1; dZ_all 192 x 1; chain no dhaux; dx_0 no dhaux, odd L'),
    'l5_s96_aux': _row(5, 96, 2, 40, [130, 1, 300, 2, 64], relu=0, aux=True,
        reaches='dWskip 1 M-block, last 96 rows, nB 5 x 2; dZ_all 64 x 5; chain with dhaux; dx_0 with dhaux, odd L'),
    'l7_s96': _row(7, 96, 2, 127, [1, 300, 2, 64, 512, 3, 130], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 96 rows, nB 7 x 2; dZ_all 64 x 7; chain no dhaux; dx_0 no dhaux, odd L'),
    'l1_s128_aux': _row(1, 128, 1, 129, [300], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 128 rows, nB 2 x 1; dZ_all 64 x 1; no chain; dx_0 with dhaux, L 1'),
    'l2_s128': _row(2, 128, 3, 63, [2, 64], relu=1, aux=False,
        reaches='dWskip 1 M-block, last 128 rows, nB 4 x 1; dZ_all 128 x 1; chain no dhaux; dx_0 no dhaux, even L'),
    'l3_s128_aux': _row(3, 128, 3, 129, [64, 512, 3], relu=1, aux=True,
        reaches='dWskip 1 M-block, last 128 rows, nB 6 x 1; dZ_all 192 x 1; chain with dhaux; dx_0 with dhaux, odd L'),
    'l5_s128': _row(5, 128, 1, 1, [512, 3, 130, 1, 300], relu=0, aux=False,
        reaches='dWskip 1 M-block, last 128 rows, nB 5 x 2; dZ_all 64 x 5; chain no dhaux; dx_0 no dhaux, odd L'),
    'l7_s128_aux': _row(7, 128, 2, 40, [3, 130, 1, 300, 2, 64, 512], relu=0, aux=True,
        reaches='dWskip 1 M-block, last 128 rows, nB 7 x 2; dZ_all 64 x 7; chain with dhaux; dx_0 with dhaux, odd L'),
    'l1_s160': _row(1, 160, 2, 127, [130], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 32 rows, nB 2 x 1, M64; dZ_all 64 x 1; no chain; dx_0 no dhaux, L 1'),
    'l2_s160_aux': _row(2, 160, 1, 129, [1, 300], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 32 rows, nB 4 x 1; dZ_all 128 x 1; chain with dhaux; dx_0 with dhaux, even L'),
    'l3_s160': _row(3, 160, 3, 63, [300, 2, 64], relu=1, aux=False,
        reaches='dWskip 2 M-blocks, last 32 rows, nB 6 x 1; dZ_all 192 x 1; chain no dhaux; dx_0 no dhaux, odd L'),
    'l5_s160_aux': _row(5, 160, 3, 129, [2, 64, 512, 3, 130], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 32 rows, nB 5 x 2; dZ_all 64 x 5; chain with dhaux; dx_0 with dhaux, odd L'),
    'l7_s160': _row(7, 160, 1, 1, [64, 512, 3, 130, 1, 300, 2], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 32 rows, nB 7 x 2; dZ_all 64 x 7; chain no dhaux; dx_0 no dhaux, odd L'),
    'l1_s192_aux': _row(1, 192, 2, 40, [512], relu=0, aux=True,
        reaches='dWskip 2 M-blocks, last 64 rows, nB 2 x 1, M64; dZ_all 64 x 1; no chain; dx_0 with dhaux, L 1'),
    'l2_s192': _row(2, 192, 2, 127, [3, 130], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 64 rows, nB 4 x 1; dZ_all 128 x 1; chain no dhaux; dx_0 no dhaux, even L'),
    'l3_s192_aux': _row(3, 192, 1, 129, [130, 1, 300], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 64 rows, nB 6 x 1; dZ_all 192 x 1; chain with dhaux; dx_0 with dhaux, odd L'),
    'l5_s192': _row(5, 192, 3, 63, [1, 300, 2, 64, 512], relu=1, aux=False,
        reaches='dWskip 2 M-blocks, last 64 rows, nB 5 x 2; dZ_all 64 x 5; chain no dhaux; dx_0 no dhaux, odd L'),
    'l7_s192_aux': _row(7, 192, 3, 129, [300, 2, 64, 512, 3, 130, 1], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 64 rows, nB 7 x 2; dZ_all 64 x 7; chain with dhaux; dx_0 with dhaux, odd L'),
    'l1_s224': _row(1, 224, 1, 1, [2], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 96 rows, nB 2 x 1; dZ_all 64 x 1; no chain; dx_0 no dhaux, L 1'),
    'l2_s224_aux': _row(2, 224, 2, 40, [64, 512], relu=0, aux=True,
        reaches='dWskip 2 M-blocks, last 96 rows, nB 4 x 1; dZ_all 128 x 1; chain with dhaux; dx_0 with dhaux, even L'),
    'l3_s224': _row(3, 224, 2, 127, [512, 3, 130], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 96 rows, nB 6 x 1; dZ_all 192 x 1; chain no dhaux; dx_0 no dhaux, odd L'),
    'l5_s224_aux': _row(5, 224, 1, 129, [3, 130, 1, 300, 2], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 96 rows, nB 5 x 2; dZ_all 64 x 5; chain with dhaux; dx_0 with dhaux, odd L'),
    'l7_s224': _row(7, 224, 3, 63, [130, 1, 300, 2, 64, 512, 3], relu=1, aux=False,
        reaches='dWskip 2 M-blocks, last 96 rows, nB 7 x 2; dZ_all 64 x 7; chain no dhaux; dx_0 no dhaux, odd L'),
    'l1_s256_aux': _row(1, 256, 3, 129, [1], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 128 rows, nB 2 x 1; dZ_all 64 x 1; no chain; dx_0 with dhaux, L 1'),
    'l2_s256': _row(2, 256, 1, 1, [300, 2], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 128 rows, nB 4 x 1; dZ_all 128 x 1; chain no dhaux; dx_0 no dhaux, even L'),
    'l3_s256_aux': _row(3, 256, 2, 40, [2, 64, 512], relu=0, aux=True,
        reaches='dWskip 2 M-blocks, last 128 rows, nB 6 x 1; dZ_all 192 x 1; chain with dhaux; dx_0 with dhaux, odd L'),
    'l5_s256': _row(5, 256, 2, 127, [64, 512, 3, 130, 1], relu=0, aux=False,
        reaches='dWskip 2 M-blocks, last 128 rows, nB 5 x 2; dZ_all 64 x 5; chain no dhaux; dx_0 no dhaux, odd L'),
    'l7_s256_aux': _row(7, 256, 1, 129, [512, 3, 130, 1, 300, 2, 64], relu=1, aux=True,
        reaches='dWskip 2 M-blocks, last 128 rows, nB 7 x 2; dZ_all 64 x 7; chain with dhaux; dx_0 with dhaux, odd L'),
    'l1_s512': _row(1, 512, 3, 63, [3], relu=1, aux=False,
        reaches='dWskip 4 M-blocks, last 128 rows, nB 2 x 1; dZ_all 64 x 1; no chain; dx_0 no dhaux, L 1'),
    'l2_s512_aux': _row(2, 512, 3, 129, [130, 1], relu=1, aux=True,
        reaches='dWskip 4 M-blocks, last 128 rows, nB 4 x 1; dZ_all 128 x 1; chain with dhaux; dx_0 with dhaux, even '
                'L'),
    'l3_s512': _row(3, 512, 1, 1, [1, 300, 2], relu=0, aux=False,
        reaches='dWskip 4 M-blocks, last 128 rows, nB 6 x 1; dZ_all 192 x 1; chain no dhaux; dx_0 no dhaux, odd L'),
    'l5_s512_aux': _row(5, 512, 2, 40, [300, 2, 64, 512, 3], relu=0, aux=True,
        reaches='dWskip 4 M-blocks, last 128 rows, nB 5 x 2; dZ_all 64 x 5; chain with dhaux; dx_0 with dhaux, odd L'),
    'l7_s512': _row(7, 512, 2, 127, [2, 64, 512, 3, 130, 1, 300], relu=0, aux=False,
        reaches='dWskip 4 M-blocks, last 128 rows, nB 7 x 2; dZ_all 64 x 7; chain no dhaux; dx_0 no dhaux, odd L'),
    # ---- the one-block dZ_all of 256 columns; weight-gradient lists of two and three launches ----
    "l4_s256": _row(4, 256, 3, 65, [5, 400, 1, 33], relu=1, aux=False,
                    reaches="dZ_all 256 x 1; chain no dhaux with a residual in both directions; dx_0 no dhaux, even L"),
    "l64_s512": _row(64, 512, 2, 40, [(29 * i) % 520 + 1 for i in range(64)], relu=1, aux=False,
                     reaches="255 weight-gradient problems: two kMaxProb launches; 64 blocks without dhaux; dZ_all "
                             "256 x 16"),
    "l59_s512_aux": _row(59, 512, 1, 100, [(53 * i) % 700 + 1 for i in range(59)], relu=0, aux=True,
                         reaches="353 weight-gradient problems: three kMaxProb launches; dWskip nB 2 x 59; dZ_all "
                                 "64 x 59"),
}

FUSED_ROWS = {
    's64': dict(S=64, d=3, B=1, T=1, last=False, init=True, aux=True,
              reaches='dW2 launches of 1 two-op M-blocks; 2 W2 chunks; dX with dhaux + dout'),
    's128': dict(S=128, d=5, B=2, T=63, last=False, init=False, aux=False,
              reaches='dW2 launches of 2 two-op M64 M-blocks; 3 W2 chunks; dX no dhaux + dout'),
    's192': dict(S=192, d=7, B=1, T=129, last=False, init=False, aux=True,
              reaches='dW2 launches of 2 two-op M-blocks; 4 W2 chunks; dX with dhaux + dout'),
    's256': dict(S=256, d=70, B=3, T=63, last=False, init=True, aux=False,
              reaches='dW2 launches of 3 two-op M64 M-blocks; 5 W2 chunks; dX no dhaux + dout'),
    's320': dict(S=320, d=64, B=2, T=65, last=False, init=True, aux=True,
              reaches='dW2 launches of 3 two-op M-blocks; 6 W2 chunks; dX with dhaux + dout'),
    's384': dict(S=384, d=2, B=3, T=129, last=False, init=False, aux=False,
              reaches='dW2 launches of 4 two-op M64 M-blocks; 7 W2 chunks; dX no dhaux + dout'),
    's448': dict(S=448, d=3, B=1, T=1, last=False, init=False, aux=True,
              reaches='dW2 launches of 4 two-op M-blocks; 8 W2 chunks; dX with dhaux + dout'),
    's512': dict(S=512, d=5, B=2, T=63, last=False, init=True, aux=False,
              reaches='dW2 launches of 5 two-op M64 M-blocks; 9 W2 chunks; dX no dhaux + dout'),
    's576': dict(S=576, d=7, B=1, T=129, last=False, init=True, aux=True,
              reaches='dW2 launches of 5 two-op M-blocks; 10 W2 chunks; dX with dhaux + dout'),
    's640': dict(S=640, d=70, B=3, T=63, last=False, init=False, aux=False,
              reaches='dW2 launches of 5 two-op + 1 M64 M-blocks; 11 W2 chunks; dX no dhaux + dout'),
    's1024': dict(S=1024, d=64, B=2, T=65, last=False, init=True, aux=True,
              reaches='dW2 launches of 5 two-op + 4 M64 M-blocks; 17 W2 chunks; dX with dhaux + dout'),
    's1152': dict(S=1152, d=2, B=3, T=129, last=False, init=False, aux=False,
              reaches='dW2 launches of 5 two-op + 5 M64 M-blocks; 19 W2 chunks; dX no dhaux + dout'),
    's128_last': dict(S=128, d=3, B=1, T=1, last=True, init=True, aux=False,
              reaches='dW2 launches of 1 M-blocks; 2 W2 chunks; dX no dhaux'),
    's192_last': dict(S=192, d=5, B=2, T=63, last=True, init=False, aux=True,
              reaches='dW2 launches of 2 M64 M-blocks; 3 W2 chunks; dX with dhaux'),
    's256_last': dict(S=256, d=7, B=1, T=129, last=True, init=False, aux=False,
              reaches='dW2 launches of 2 M-blocks; 4 W2 chunks; dX no dhaux'),
    's320_last': dict(S=320, d=70, B=3, T=63, last=True, init=True, aux=True,
              reaches='dW2 launches of 3 M64 M-blocks; 5 W2 chunks; dX with dhaux'),
    's512_last': dict(S=512, d=64, B=2, T=65, last=True, init=True, aux=False,
              reaches='dW2 launches of 4 M-blocks; 8 W2 chunks; dX no dhaux'),
    's1024_last': dict(S=1024, d=2, B=3, T=129, last=True, init=False, aux=True,
              reaches='dW2 launches of 5 + 3 M-blocks; 16 W2 chunks; dX with dhaux'),
}

# the launch variants of the coverage grid (tests/test_stack_shapes_host.py), stack and fused path
STACK_VARIANTS = 82
FUSED_VARIANTS = 35
