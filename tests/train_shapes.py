# -*- coding: utf-8 -*-
"""The shape table of tests/test_gpu_train_shapes.py and tests/test_train_shapes_host.py: the per-block tensor-core
training path (``resblock_fwd_composed`` and the composed branch of ``wnb_resblock_bwd``) and the tensor-core post
network, across their whole coverage.

``composed_tc_supported(R, S, Ap, ks)`` covers R in {64, 128, 192, 256, 512}, S in {32, 64, ..., 256, 512}, Ap in
{32, 64, ..., 256} and ks in {1, 2, 3}: 1 080 shapes, every one of them in bf16 and all but the five that the fused
R = 64 kernel takes in tf32.  Each launch of the path is a template instantiation or a split of the work that depends
on the shape (tests/test_train_shapes_host.py restates the dispatch and names them); the rows together reach every one
that the coverage grid reaches, in both modes.  The R x Ap pairs form a full 5 x 8 grid (the haux weight gradient's
M-block count and column split); ks cycles so that every R meets every ks and every Ap meets ks 3; S and ``last`` are
chosen per R so that the rows reach every M-block count, launch split, a0 | a1 straddle and M = 64 form of the
res/skip weight gradient.

Block rows: ``R, S, Ap, ks`` the block shape, ``d`` its dilation, ``B, T`` the batch, ``last`` dout is NULL (no xout,
no res GEMM, only the skip rows of dW2), ``init`` skip is stored rather than accumulated, ``modes`` the math modes that
run the row on the composed path (tf32 leaves R = 64, ks 2, Ap 32 with S a multiple of 64 to the fused kernel),
``tf32_bwd`` which tf32 backward an R = 64 row takes ("composed", or "r64": the R = 64 gate-GEMM backward of
``tc_fused_shape``, R == 64 && ks == 2 && Ap == 32 && S % 32 == 0), and ``reaches`` what the row is there for.
Time profiles cycle through T = 1, T one under and one over a multiple of 64, odd 64-row tile counts over B = 1 and 3
(the last CTA of a two-tile pair half empty, pairs spanning utterances) and d >= T.

Post rows: ``S, Q, B, T``, ``rectified`` (``skip_rectified``: 0 = the forward rectifies skip in place) and ``modes``.
Per S every class of Q that changes the dWp2 launch: Q <= 64 (one M-block, the M = 64 form when nB <= 3), 96 / 128
(one full M-block), 160..256 (two) and 512 (four, and the N = 512 logits GEMM in two column blocks)."""
BOTH = ("tf32", "bf16")

BLOCK_ROWS = {
    # ---- R = 64 ----
    "r64_s32_a32_k1": dict(R=64, S=32, Ap=32, ks=1, d=3, B=2, T=65, last=False, init=True, modes=BOTH,
                           tf32_bwd="composed",
                           reaches="1 gate launch of 64; dhaux N 32, dW1 aux nB 1 x 1; dW2 1 M-block, straddling "
                                   "a0|a1; xout/dx add via TMA"),
    "r64_s96_a64_k2_last": dict(R=64, S=96, Ap=64, ks=2, d=1, B=1, T=1, last=True, init=False, modes=BOTH,
                                tf32_bwd="composed",
                                reaches="1 gate launch of 64; dhaux N 64, dW1 aux nB 2 x 1; dW2 1 M-block"),
    "r64_s512_a96_k3": dict(R=64, S=512, Ap=96, ks=3, d=5, B=3, T=63, last=False, init=True, modes=BOTH,
                            tf32_bwd="composed",
                            reaches="1 gate launch of 64; dhaux N 96, dW1 aux nB 3 x 1; dW2 5 M-blocks, straddling "
                                    "a0|a1, M64; skip in 2 blocks; xout/dx add via TMA"),
    "r64_s160_a128_k1_last": dict(R=64, S=160, Ap=128, ks=1, d=64, B=3, T=129, last=True, init=False, modes=BOTH,
                                  tf32_bwd="composed",
                                  reaches="1 gate launch of 64; dhaux N 128, dW1 aux nB 4 x 1; dW2 2 M-blocks, M64"),
    "r64_s256_a160_k2": dict(R=64, S=256, Ap=160, ks=2, d=128, B=2, T=100, last=False, init=True, modes=BOTH,
                             tf32_bwd="composed",
                             reaches="1 gate launch of 64; dhaux N 160, dW1 aux nB 1 x 5; dW2 3 M-blocks, straddling "
                                     "a0|a1, M64; xout/dx add via TMA"),
    "r64_s64_a192_k3_last": dict(R=64, S=64, Ap=192, ks=3, d=7, B=1, T=191, last=True, init=False, modes=BOTH,
                                 tf32_bwd="composed",
                                 reaches="1 gate launch of 64; dhaux N 192, dW1 aux nB 3 x 2; dW2 1 M-block, M64"),
    "r64_s192_a224_k1": dict(R=64, S=192, Ap=224, ks=1, d=2, B=2, T=33, last=False, init=True, modes=BOTH,
                             tf32_bwd="composed",
                             reaches="1 gate launch of 64; dhaux N 224, dW1 aux nB 1 x 7; dW2 2 M-blocks, straddling "
                                     "a0|a1; xout/dx add via TMA"),
    "r64_s512_a256_k2_last": dict(R=64, S=512, Ap=256, ks=2, d=3, B=2, T=65, last=True, init=False, modes=BOTH,
                                  tf32_bwd="composed",
                                  reaches="1 gate launch of 64; dhaux N 256, dW1 aux nB 4 x 2; dW2 4 M-blocks; skip "
                                          "in 2 blocks"),
    "r64_s224_a96_k2_last": dict(R=64, S=224, Ap=96, ks=2, d=1, B=1, T=1, last=True, init=True, modes=BOTH,
                                 tf32_bwd="composed",
                                 reaches="1 gate launch of 64; dhaux N 96, dW1 aux nB 3 x 1; dW2 2 M-blocks"),
    "r64_s128_a64_k3": dict(R=64, S=128, Ap=64, ks=3, d=5, B=3, T=63, last=False, init=False, modes=BOTH,
                            tf32_bwd="composed",
                            reaches="1 gate launch of 64; dhaux N 64, dW1 aux nB 2 x 1; dW2 2 M-blocks, straddling "
                                    "a0|a1, M64; xout/dx add via TMA"),
    # ---- R = 128 ----
    "r128_s256_a32_k2": dict(R=128, S=256, Ap=32, ks=2, d=64, B=3, T=129, last=False, init=True, modes=BOTH,
                             reaches="1 gate launch of 128; dhaux N 32, dW1 aux nB 1 x 1; dW2 3 M-blocks; xout/dx add "
                                     "via __ldg"),
    "r128_s32_a64_k3_last": dict(R=128, S=32, Ap=64, ks=3, d=128, B=2, T=100, last=True, init=False, modes=BOTH,
                                 reaches="1 gate launch of 128; dhaux N 64, dW1 aux nB 2 x 1; dW2 1 M-block"),
    "r128_s512_a96_k1_last": dict(R=128, S=512, Ap=96, ks=1, d=7, B=1, T=191, last=True, init=True, modes=BOTH,
                                  reaches="1 gate launch of 128; dhaux N 96, dW1 aux nB 3 x 1; dW2 4 M-blocks; skip "
                                          "in 2 blocks"),
    "r128_s96_a128_k2": dict(R=128, S=96, Ap=128, ks=2, d=2, B=2, T=33, last=False, init=False, modes=BOTH,
                             reaches="1 gate launch of 128; dhaux N 128, dW1 aux nB 4 x 1; dW2 2 M-blocks; xout/dx "
                                     "add via __ldg"),
    "r128_s512_a160_k3": dict(R=128, S=512, Ap=160, ks=3, d=3, B=2, T=65, last=False, init=True, modes=BOTH,
                              reaches="1 gate launch of 128; dhaux N 160, dW1 aux nB 1 x 5; dW2 5 M-blocks; skip in 2 "
                                      "blocks; xout/dx add via __ldg"),
    "r128_s224_a192_k1_last": dict(R=128, S=224, Ap=192, ks=1, d=1, B=1, T=1, last=True, init=False, modes=BOTH,
                                   reaches="1 gate launch of 128; dhaux N 192, dW1 aux nB 3 x 2; dW2 2 M-blocks"),
    "r128_s160_a224_k2": dict(R=128, S=160, Ap=224, ks=2, d=5, B=3, T=63, last=False, init=True, modes=BOTH,
                              reaches="1 gate launch of 128; dhaux N 224, dW1 aux nB 1 x 7; dW2 3 M-blocks; xout/dx "
                                      "add via __ldg"),
    "r128_s128_a256_k3_last": dict(R=128, S=128, Ap=256, ks=3, d=64, B=3, T=129, last=True, init=False, modes=BOTH,
                                   reaches="1 gate launch of 128; dhaux N 256, dW1 aux nB 4 x 2; dW2 1 M-block"),
    # ---- R = 192 ----
    "r192_s64_a32_k3": dict(R=192, S=64, Ap=32, ks=3, d=128, B=2, T=100, last=False, init=True, modes=BOTH,
                            reaches="3 gate launches of 64; dhaux N 32, dW1 aux nB 1 x 1; dW2 2 M-blocks, straddling "
                                    "a0|a1; xout/dx add via __ldg"),
    "r192_s128_a64_k1_last": dict(R=192, S=128, Ap=64, ks=1, d=7, B=1, T=191, last=True, init=False, modes=BOTH,
                                  reaches="3 gate launches of 64; dhaux N 64, dW1 aux nB 2 x 1; dW2 1 M-block"),
    "r192_s512_a96_k2": dict(R=192, S=512, Ap=96, ks=2, d=2, B=2, T=33, last=False, init=True, modes=BOTH,
                             reaches="3 gate launches of 64; dhaux N 96, dW1 aux nB 3 x 1; dW2 6 M-blocks 3+3, "
                                     "straddling a0|a1, M64; skip in 2 blocks; xout/dx add via __ldg"),
    "r192_s32_a128_k3_last": dict(R=192, S=32, Ap=128, ks=3, d=3, B=2, T=65, last=True, init=False, modes=BOTH,
                                  reaches="3 gate launches of 64; dhaux N 128, dW1 aux nB 4 x 1; dW2 1 M-block, M64"),
    "r192_s256_a160_k1_last": dict(R=192, S=256, Ap=160, ks=1, d=1, B=1, T=1, last=True, init=True, modes=BOTH,
                                   reaches="3 gate launches of 64; dhaux N 160, dW1 aux nB 1 x 5; dW2 2 M-blocks"),
    "r192_s192_a192_k2": dict(R=192, S=192, Ap=192, ks=2, d=5, B=3, T=63, last=False, init=False, modes=BOTH,
                              reaches="3 gate launches of 64; dhaux N 192, dW1 aux nB 3 x 2; dW2 3 M-blocks, "
                                      "straddling a0|a1; xout/dx add via __ldg"),
    "r192_s96_a224_k3": dict(R=192, S=96, Ap=224, ks=3, d=64, B=3, T=129, last=False, init=True, modes=BOTH,
                             reaches="3 gate launches of 64; dhaux N 224, dW1 aux nB 1 x 7; dW2 3 M-blocks, "
                                     "straddling a0|a1, M64; xout/dx add via __ldg"),
    "r192_s512_a256_k1_last": dict(R=192, S=512, Ap=256, ks=1, d=128, B=2, T=100, last=True, init=False, modes=BOTH,
                                   reaches="3 gate launches of 64; dhaux N 256, dW1 aux nB 4 x 2; dW2 4 M-blocks; "
                                           "skip in 2 blocks"),
    "r192_s160_a160_k2_last": dict(R=192, S=160, Ap=160, ks=2, d=7, B=1, T=191, last=True, init=True, modes=BOTH,
                                   reaches="3 gate launches of 64; dhaux N 160, dW1 aux nB 1 x 5; dW2 2 M-blocks, M64"),
    "r192_s224_a224_k1": dict(R=192, S=224, Ap=224, ks=1, d=2, B=2, T=33, last=False, init=False, modes=BOTH,
                              reaches="3 gate launches of 64; dhaux N 224, dW1 aux nB 1 x 7; dW2 4 M-blocks, "
                                      "straddling a0|a1, M64; xout/dx add via __ldg"),
    # ---- R = 256 ----
    "r256_s96_a32_k1_last": dict(R=256, S=96, Ap=32, ks=1, d=3, B=2, T=65, last=True, init=True, modes=BOTH,
                                 reaches="2 gate launches of 128; dhaux N 32, dW1 aux nB 1 x 1; dW2 1 M-block"),
    "r256_s192_a64_k2_last": dict(R=256, S=192, Ap=64, ks=2, d=1, B=1, T=1, last=True, init=False, modes=BOTH,
                                  reaches="2 gate launches of 128; dhaux N 64, dW1 aux nB 2 x 1; dW2 2 M-blocks"),
    "r256_s64_a96_k3": dict(R=256, S=64, Ap=96, ks=3, d=5, B=3, T=63, last=False, init=True, modes=BOTH,
                            reaches="2 gate launches of 128; dhaux N 96, dW1 aux nB 3 x 1; dW2 3 M-blocks; xout/dx "
                                    "add via __ldg"),
    "r256_s512_a128_k1": dict(R=256, S=512, Ap=128, ks=1, d=64, B=3, T=129, last=False, init=False, modes=BOTH,
                              reaches="2 gate launches of 128; dhaux N 128, dW1 aux nB 4 x 1; dW2 6 M-blocks 3+3; "
                                      "skip in 2 blocks; xout/dx add via __ldg"),
    "r256_s224_a160_k2": dict(R=256, S=224, Ap=160, ks=2, d=128, B=2, T=100, last=False, init=True, modes=BOTH,
                              reaches="2 gate launches of 128; dhaux N 160, dW1 aux nB 1 x 5; dW2 4 M-blocks; xout/dx "
                                      "add via __ldg"),
    "r256_s160_a192_k3": dict(R=256, S=160, Ap=192, ks=3, d=7, B=1, T=191, last=False, init=False, modes=BOTH,
                              reaches="2 gate launches of 128; dhaux N 192, dW1 aux nB 3 x 2; dW2 4 M-blocks; xout/dx "
                                      "add via __ldg"),
    "r256_s512_a224_k1_last": dict(R=256, S=512, Ap=224, ks=1, d=2, B=2, T=33, last=True, init=True, modes=BOTH,
                                   reaches="2 gate launches of 128; dhaux N 224, dW1 aux nB 1 x 7; dW2 4 M-blocks; "
                                           "skip in 2 blocks"),
    "r256_s32_a256_k2": dict(R=256, S=32, Ap=256, ks=2, d=3, B=2, T=65, last=False, init=False, modes=BOTH,
                             reaches="2 gate launches of 128; dhaux N 256, dW1 aux nB 4 x 2; dW2 3 M-blocks; xout/dx "
                                     "add via __ldg"),
    # ---- R = 512 ----
    "r512_s512_a32_k2": dict(R=512, S=512, Ap=32, ks=2, d=1, B=1, T=1, last=False, init=True, modes=BOTH,
                             reaches="4 gate launches of 128; dhaux N 32, dW1 aux nB 1 x 1; dW2 8 M-blocks 4+4; skip "
                                     "in 2 blocks; res/dz/dx in 2 blocks; xout/dx add via __ldg"),
    "r512_s128_a64_k3_last": dict(R=512, S=128, Ap=64, ks=3, d=5, B=3, T=63, last=True, init=False, modes=BOTH,
                                  reaches="4 gate launches of 128; dhaux N 64, dW1 aux nB 2 x 1; dW2 1 M-block; "
                                          "res/dz/dx in 2 blocks"),
    "r512_s256_a96_k1": dict(R=512, S=256, Ap=96, ks=1, d=64, B=3, T=129, last=False, init=True, modes=BOTH,
                             reaches="4 gate launches of 128; dhaux N 96, dW1 aux nB 3 x 1; dW2 6 M-blocks 3+3; "
                                     "res/dz/dx in 2 blocks; xout/dx add via __ldg"),
    "r512_s32_a128_k2": dict(R=512, S=32, Ap=128, ks=2, d=128, B=2, T=100, last=False, init=False, modes=BOTH,
                             reaches="4 gate launches of 128; dhaux N 128, dW1 aux nB 4 x 1; dW2 5 M-blocks; "
                                     "res/dz/dx in 2 blocks; xout/dx add via __ldg"),
    "r512_s192_a160_k3_last": dict(R=512, S=192, Ap=160, ks=3, d=7, B=1, T=191, last=True, init=True, modes=BOTH,
                                   reaches="4 gate launches of 128; dhaux N 160, dW1 aux nB 1 x 5; dW2 2 M-blocks; "
                                           "res/dz/dx in 2 blocks"),
    "r512_s512_a192_k1_last": dict(R=512, S=512, Ap=192, ks=1, d=2, B=2, T=33, last=True, init=False, modes=BOTH,
                                   reaches="4 gate launches of 128; dhaux N 192, dW1 aux nB 3 x 2; dW2 4 M-blocks; "
                                           "skip in 2 blocks; res/dz/dx in 2 blocks"),
    "r512_s160_a224_k2": dict(R=512, S=160, Ap=224, ks=2, d=3, B=2, T=65, last=False, init=True, modes=BOTH,
                              reaches="4 gate launches of 128; dhaux N 224, dW1 aux nB 1 x 7; dW2 6 M-blocks 3+3; "
                                      "res/dz/dx in 2 blocks; xout/dx add via __ldg"),
    "r512_s224_a256_k3_last": dict(R=512, S=224, Ap=256, ks=3, d=1, B=1, T=1, last=True, init=False, modes=BOTH,
                                   reaches="4 gate launches of 128; dhaux N 256, dW1 aux nB 4 x 2; dW2 2 M-blocks; "
                                           "res/dz/dx in 2 blocks"),
    # ---- R = 64, ks 2, Ap 32: the forward is composed, the tf32 backward is the R = 64 gate-GEMM path ----
    "r64_s96_a32_k2_r64bwd": dict(R=64, S=96, Ap=32, ks=2, d=70, B=2, T=65, last=False, init=False, modes=BOTH,
                                  tf32_bwd="r64",
                                  reaches="tf32: composed forward with the R = 64 gate-GEMM backward"),
    # ---- tf32 runs this shape on the fused kernel: bf16 only ----
    "r64_s128_a32_k2_bf16": dict(R=64, S=128, Ap=32, ks=2, d=4, B=3, T=129, last=False, init=True, modes=('bf16',),
                                 reaches="bf16 at a shape the tf32 fused kernel takes"),
}

POST_ROWS = {
    "s32_q32": dict(S=32, Q=32, B=1, T=1, rectified=0, modes=BOTH,
                    reaches="dWp2 1 M-block (last 32 rows) nB 1 x 1, M64; dWp1 nB 1 x 1, M64"),
    "s32_q96": dict(S=32, Q=96, B=2, T=65, rectified=1, modes=BOTH,
                    reaches="dWp2 1 M-block (last 96 rows) nB 1 x 1; dWp1 nB 1 x 1, M64"),
    "s32_q160": dict(S=32, Q=160, B=3, T=63, rectified=0, modes=BOTH,
                     reaches="dWp2 2 M-blocks (last 32 rows) nB 1 x 1, M64; dWp1 nB 1 x 1, M64"),
    "s32_q224": dict(S=32, Q=224, B=1, T=130, rectified=1, modes=BOTH,
                     reaches="dWp2 2 M-blocks (last 96 rows) nB 1 x 1; dWp1 nB 1 x 1, M64"),
    "s32_q512": dict(S=32, Q=512, B=2, T=31, rectified=0, modes=BOTH,
                     reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 1 x 1; dWp1 nB 1 x 1, M64"),
    "s64_q64": dict(S=64, Q=64, B=1, T=1, rectified=1, modes=BOTH,
                    reaches="dWp2 1 M-block (last 64 rows) nB 2 x 1, M64; dWp1 nB 2 x 1, M64"),
    "s64_q128": dict(S=64, Q=128, B=2, T=65, rectified=0, modes=BOTH,
                     reaches="dWp2 1 M-block nB 2 x 1; dWp1 nB 2 x 1, M64"),
    "s64_q192": dict(S=64, Q=192, B=3, T=63, rectified=1, modes=BOTH,
                     reaches="dWp2 2 M-blocks (last 64 rows) nB 2 x 1, M64; dWp1 nB 2 x 1, M64"),
    "s64_q256": dict(S=64, Q=256, B=1, T=130, rectified=0, modes=BOTH,
                     reaches="dWp2 2 M-blocks nB 2 x 1; dWp1 nB 2 x 1, M64"),
    "s64_q512": dict(S=64, Q=512, B=2, T=31, rectified=1, modes=BOTH,
                     reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 2 x 1; dWp1 nB 2 x 1, M64"),
    "s96_q32": dict(S=96, Q=32, B=1, T=1, rectified=0, modes=BOTH,
                    reaches="dWp2 1 M-block (last 32 rows) nB 3 x 1, M64; dWp1 nB 3 x 1"),
    "s96_q96": dict(S=96, Q=96, B=2, T=65, rectified=1, modes=BOTH,
                    reaches="dWp2 1 M-block (last 96 rows) nB 3 x 1; dWp1 nB 3 x 1"),
    "s96_q160": dict(S=96, Q=160, B=3, T=63, rectified=0, modes=BOTH,
                     reaches="dWp2 2 M-blocks (last 32 rows) nB 3 x 1, M64; dWp1 nB 3 x 1"),
    "s96_q224": dict(S=96, Q=224, B=1, T=130, rectified=1, modes=BOTH,
                     reaches="dWp2 2 M-blocks (last 96 rows) nB 3 x 1; dWp1 nB 3 x 1"),
    "s96_q512": dict(S=96, Q=512, B=2, T=31, rectified=0, modes=BOTH,
                     reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 3 x 1; dWp1 nB 3 x 1"),
    "s128_q64": dict(S=128, Q=64, B=1, T=1, rectified=1, modes=BOTH,
                     reaches="dWp2 1 M-block (last 64 rows) nB 4 x 1; dWp1 nB 4 x 1"),
    "s128_q256": dict(S=128, Q=256, B=2, T=65, rectified=0, modes=BOTH,
                      reaches="dWp2 2 M-blocks nB 4 x 1; dWp1 nB 4 x 1"),
    "s128_q512": dict(S=128, Q=512, B=3, T=63, rectified=1, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 4 x 1; dWp1 nB 4 x 1"),
    "s160_q32": dict(S=160, Q=32, B=1, T=130, rectified=0, modes=BOTH,
                     reaches="dWp2 1 M-block (last 32 rows) nB 1 x 5, M64; dWp1 nB 1 x 5, M64"),
    "s160_q128": dict(S=160, Q=128, B=2, T=31, rectified=1, modes=BOTH,
                      reaches="dWp2 1 M-block nB 1 x 5; dWp1 nB 1 x 5, M64"),
    "s160_q160": dict(S=160, Q=160, B=1, T=1, rectified=0, modes=BOTH,
                      reaches="dWp2 2 M-blocks (last 32 rows) nB 1 x 5, M64; dWp1 nB 1 x 5, M64"),
    "s160_q256": dict(S=160, Q=256, B=2, T=65, rectified=1, modes=BOTH,
                      reaches="dWp2 2 M-blocks nB 1 x 5; dWp1 nB 1 x 5, M64"),
    "s160_q512": dict(S=160, Q=512, B=3, T=63, rectified=0, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 1 x 5; dWp1 nB 1 x 5, M64"),
    "s192_q64": dict(S=192, Q=64, B=1, T=130, rectified=1, modes=BOTH,
                     reaches="dWp2 1 M-block (last 64 rows) nB 3 x 2, M64; dWp1 nB 3 x 2, M64"),
    "s192_q96": dict(S=192, Q=96, B=2, T=31, rectified=0, modes=BOTH,
                     reaches="dWp2 1 M-block (last 96 rows) nB 3 x 2; dWp1 nB 3 x 2, M64"),
    "s192_q192": dict(S=192, Q=192, B=1, T=1, rectified=1, modes=BOTH,
                      reaches="dWp2 2 M-blocks (last 64 rows) nB 3 x 2, M64; dWp1 nB 3 x 2, M64"),
    "s192_q256": dict(S=192, Q=256, B=2, T=65, rectified=0, modes=BOTH,
                      reaches="dWp2 2 M-blocks nB 3 x 2; dWp1 nB 3 x 2, M64"),
    "s192_q512": dict(S=192, Q=512, B=3, T=63, rectified=1, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 3 x 2; dWp1 nB 3 x 2, M64"),
    "s224_q32": dict(S=224, Q=32, B=1, T=130, rectified=0, modes=BOTH,
                     reaches="dWp2 1 M-block (last 32 rows) nB 1 x 7, M64; dWp1 nB 1 x 7"),
    "s224_q128": dict(S=224, Q=128, B=2, T=31, rectified=1, modes=BOTH,
                      reaches="dWp2 1 M-block nB 1 x 7; dWp1 nB 1 x 7"),
    "s224_q192": dict(S=224, Q=192, B=1, T=1, rectified=0, modes=BOTH,
                      reaches="dWp2 2 M-blocks (last 64 rows) nB 1 x 7, M64; dWp1 nB 1 x 7"),
    "s224_q224": dict(S=224, Q=224, B=2, T=65, rectified=1, modes=BOTH,
                      reaches="dWp2 2 M-blocks (last 96 rows) nB 1 x 7; dWp1 nB 1 x 7"),
    "s224_q512": dict(S=224, Q=512, B=3, T=63, rectified=0, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 1 x 7; dWp1 nB 1 x 7"),
    "s256_q96": dict(S=256, Q=96, B=1, T=130, rectified=1, modes=BOTH,
                     reaches="dWp2 1 M-block (last 96 rows) nB 4 x 2; dWp1 nB 4 x 2"),
    "s256_q224": dict(S=256, Q=224, B=2, T=31, rectified=0, modes=BOTH,
                      reaches="dWp2 2 M-blocks (last 96 rows) nB 4 x 2; dWp1 nB 4 x 2"),
    "s256_q512": dict(S=256, Q=512, B=1, T=1, rectified=1, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; dWp2 4 M-blocks nB 4 x 2; dWp1 nB 4 x 2"),
    "s512_q32": dict(S=512, Q=32, B=2, T=65, rectified=0, modes=BOTH,
                     reaches="post_split; dWp2 1 M-block (last 32 rows) nB 4 x 4; dWp1 nB 4 x 4"),
    "s512_q256": dict(S=512, Q=256, B=3, T=63, rectified=1, modes=BOTH,
                      reaches="post_split; dWp2 2 M-blocks nB 4 x 4; dWp1 nB 4 x 4"),
    "s512_q512": dict(S=512, Q=512, B=1, T=130, rectified=0, modes=BOTH,
                      reaches="logits N 512 in 2 blocks; post_split; dWp2 4 M-blocks nB 4 x 4; dWp1 nB 4 x 4"),
}
