# -*- coding: utf-8 -*-
"""CPU tier: the training shape table (tests/train_shapes.py) reaches the whole coverage of the per-block tensor-core
path and of the tensor-core post network, from the library's coverage queries and from a restatement of their dispatch.

* every block row takes the forward the table claims (``wnb_resblock_fwd_supported``: 2 composed, 1 fused) in tf32,
  and the composed path in bf16; every R = 64 row names the tf32 backward it takes;
* over a grid that contains the whole coverage (R, S in 32..1 024, Ap in 32..512, ks 1..4, ``last`` both ways) the
  library's predicate is exactly ``composed_tc_supported``, the rows reach every value of every axis, and the launch
  variants of the rows are exactly the launch variants of the grid -- in tf32 and in bf16;
* the post rows' launch variants are those of every (S, Q) the post network's tensor-core branch takes, with
  ``skip_rectified`` both ways;
* ``nets.wavenet.bf16_supported`` agrees with the library over the grid with Q in 32..1 024.

A launch variant is what one launch of the path instantiates or how it splits its work: for ``gemm_nt_tc`` the role,
N, the epilogue, the operand type, the column blocks and how the epilogue's add operand is read (TMA, ``__ldg`` or
none), and for the gate GEMMs the number of launches; for ``wgrad_tc_concat`` the role, the M-block count and its split
over launches, nB, the all-ones bias group, n_split, whether an M-block straddles the a0 | a1 concatenation and whether
the kernel runs its M = 64 form.  A new instantiation or split that no row reaches makes the set equality fail."""
import itertools

import pytest

from pytorchwavenetvocoder_b200 import _lib
from tests import train_shapes as TS

MODES = ("tf32", "bf16")
GRID_RS = range(32, 1025, 32)
GRID_AP = range(32, 513, 32)
GRID_KS = (1, 2, 3, 4)
GRID_Q = range(32, 1025, 32)
R_ALL = (64, 128, 192, 256, 512)
S_ALL = (32, 64, 96, 128, 160, 192, 224, 256, 512)
AP_ALL = (32, 64, 96, 128, 160, 192, 224, 256)
KS_ALL = (1, 2, 3)


# ------------------------------------------------------------------------------------------------------------------
# the dispatch, restated (csrc/resblock_simt.cu, csrc/gemm_nt_tc.cu, csrc/wgrad_tc.cu, csrc/resblock_z.cu)
# ------------------------------------------------------------------------------------------------------------------
def nt_tc_n_ok(N):
    """resblock_simt.cu:405 nt_tc_n_ok"""
    return N % 32 == 0 and N >= 32 and (N <= 256 or N == 512)


def composed_tc_supported(R, S, Ap, ks):
    """resblock_simt.cu:574-576 composed_tc_supported"""
    return R % 64 == 0 and nt_tc_n_ok(R) and nt_tc_n_ok(S) and Ap % 32 == 0 and Ap <= 256 and 1 <= ks <= 3


def fused_fwd(R, S, Ap, ks):
    """resblock_z.cu:496-498 resblock_fwd_skip_supported: the fused R = 64 forward (tf32 only)"""
    return R == 64 and ks == 2 and Ap == 32 and S >= 64 and S % 64 == 0


def tc_fused_bwd(R, S, Ap, ks):
    """resblock_simt.cu:719 tc_fused_shape: the R = 64 gate-GEMM backward (tf32 only) -- not the forward's rule"""
    return R == 64 and ks == 2 and Ap == 32 and S % 32 == 0


def composed_gc(R):
    """resblock_simt.cu:579 composed_gc: gate channels per gate GEMM"""
    return 128 if R % 128 == 0 else 64


def plain_nblk(N):
    """resblock_simt.cu:580-584 plain_opts: column blocks of the plain composed GEMMs"""
    return N // 256 if (N > 256 and N % 256 == 0) else 1


def post_split(S):
    """resblock_simt.cu:399-403 post_split (WNB_POST_SPLIT unset)"""
    return S == 512


def gemm(role, op, N, epi="plain", nblk=1, add=None, launches=1):
    """gemm_nt_tc.cu:547-554: N = 512 runs as two 256-column blocks.  gemm_nt_tc.cu:627-640: the plain epilogue's add
    operand goes through TMA when add_cols (= N) <= 32 kMaxEop (= 64, gemm_nt_tc.cu:58) and is 16-byte aligned (every
    operand here is), through __ldg otherwise; the gate backward's dz goes through TMA at 64 gate channels
    (``add`` = "dz")."""
    if N == 512:
        N, nblk = 256, 2
    if add is None:
        how = "none"
    elif add == "dz":
        how = "tma" if N // 2 == 64 else "ldg"
    else:
        how = "tma" if N <= 64 else "ldg"        # add_cols = N: none of these GEMMs has a split output
    return ("gemm", role, op, N, epi, nblk, how, launches)


def wgrad_concat(role, op, C0, has_a1, M, N, db):
    """resblock_simt.cu:522-571 wgrad_tc_concat and the problem list of wgrad_tc.cu:516-592 it feeds"""
    groups = N // 32
    nB = next(g for g in (4, 3, 2, 1) if groups % g == 0 and groups // g <= 128)      # :532-534
    mblocks = (M + 127) // 128                                                        # :535-539
    launches = (mblocks + 4) // 5
    per = (mblocks + launches - 1) // launches
    split = tuple(min(per, mblocks - i) for i in range(0, mblocks, per))
    n_split = groups // nB                                                             # :540
    ones = 1 if db else 0                                                              # wgrad_tc.cu:519-521
    m_last = M - (mblocks - 1) * 128                                                   # :548
    straddle = has_a1 and C0 % 128 != 0 and C0 < M                                   # :558-563
    m64 = m_last <= 64 and 32 * (nB + ones) <= 128                                    # wgrad_tc.cu:544 pr.nA
    return ("wgrad", role, op, mblocks, split, nB, ones, n_split, straddle, m64)


def block_variants(R, S, Ap, ks, last, mode):
    """the launches of one composed block: resblock_fwd_composed (resblock_simt.cu:590-619) and the composed branch of
    wnb_resblock_bwd (resblock_simt.cu:719-781), or the R = 64 gate-GEMM backward (:782-871) in tf32"""
    assert composed_tc_supported(R, S, Ap, ks) and not (mode == "tf32" and fused_fwd(R, S, Ap, ks))
    op = mode
    GC = composed_gc(R)
    v = {gemm("gate_fwd", op, 2 * GC, "gate", launches=R // GC)}                        # :599-605
    if not last:                                                                       # :606-613 (xout)
        v.add(gemm("res", op, R // plain_nblk(R), nblk=plain_nblk(R), add="xin"))
    v.add(gemm("skip", op, S // plain_nblk(S), nblk=plain_nblk(S)))                     # :614-618
    if mode == "tf32" and tc_fused_bwd(R, S, Ap, ks):                                  # :719-721, :782-871
        v.add(("r64_bwd", op))
        return v
    nb = plain_nblk(R)                                                                 # :732
    v.add(gemm("dz", op, R // nb, nblk=nb))                                            # :733-745
    v.add(gemm("gate_bwd", op, 2 * GC, "gate", add="dz", launches=R // GC))             # :751-757
    v.add(gemm("dx", op, R // nb, nblk=nb, add=None if last else "dout"))              # :758-765
    v.add(gemm("dhaux", op, Ap))                                                       # :766-770
    for j in range(ks):                                                                # :772-775
        v.add(wgrad_concat("dW1_tap0" if j == 0 else "dW1_tap", op, 2 * R, False, 2 * R, R, j == 0))
    v.add(wgrad_concat("dW1_aux", op, 2 * R, False, 2 * R, Ap, False))                  # :776-778
    if last:                                                                           # :780
        v.add(wgrad_concat("dW2", op, S, False, S, R, True))
    else:                                                                              # :779
        v.add(wgrad_concat("dW2", op, R, True, R + S, R, True))
    return v


def post_variants(S, Q, rectified, mode):
    """the tensor-core branches of wnb_post_fwd (resblock_simt.cu:910-937) and wnb_post_bwd (:968-1005)"""
    assert nt_tc_n_ok(S) and nt_tc_n_ok(Q)
    op = mode
    v = set()
    if not rectified:                                                                  # :920-923
        v.add(("relu_inplace",))
    nb = 2 if post_split(S) else 1                                                     # :926-931, :980-991
    v.add(gemm("post1", op, S // nb, nblk=nb))
    v.add(gemm("post2", op, Q))                                                        # :932-936
    v.add(gemm("post_dh1", op, S // nb, nblk=nb))
    v.add(gemm("post_dskip", op, S // nb, nblk=nb))
    v.add(wgrad_concat("dWp2", op, Q, False, Q, S, True))                               # :996 / :1003
    v.add(wgrad_concat("dWp1", op, S, False, S, S, True))                               # :997 / :1004
    return v


def row_modes(R, S, Ap, ks):
    """the modes that run a shape on the composed path"""
    if not composed_tc_supported(R, S, Ap, ks):
        return ()
    return ("bf16",) if fused_fwd(R, S, Ap, ks) else MODES


def _block_grid():
    for R, S, Ap, ks in itertools.product(GRID_RS, GRID_RS, GRID_AP, GRID_KS):
        yield R, S, Ap, ks


def _shape(row):
    return row["R"], row["S"], row["Ap"], row["ks"]


# ------------------------------------------------------------------------------------------------------------------
# the rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rid", list(TS.BLOCK_ROWS))
def test_block_row_takes_the_path_it_claims(rid):
    row = TS.BLOCK_ROWS[rid]
    lib = _lib.load()
    R, S, Ap, ks = _shape(row)
    assert row["modes"] and set(row["modes"]) <= set(MODES), rid
    assert tuple(row["modes"]) == row_modes(R, S, Ap, ks), rid
    assert lib.wnb_resblock_fwd_supported(R, S, Ap, ks, _lib.MATH_TF32) == (2 if "tf32" in row["modes"] else 1), rid
    assert "bf16" in row["modes"] and lib.wnb_resblock_fwd_supported(R, S, Ap, ks, _lib.MATH_BF16) == 2, rid
    # the tf32 backward: R = 64 rows say which one they take
    if R == 64 and "tf32" in row["modes"]:
        assert row["tf32_bwd"] == ("r64" if tc_fused_bwd(R, S, Ap, ks) else "composed"), rid
    else:
        assert row.get("tf32_bwd") in (None, "composed"), rid
    assert row["B"] >= 1 and row["T"] >= 1 and row["d"] >= 1 and row["reaches"], rid


@pytest.mark.parametrize("rid", list(TS.POST_ROWS))
def test_post_row_takes_the_tensor_core_branch(rid):
    row = TS.POST_ROWS[rid]
    assert nt_tc_n_ok(row["S"]) and nt_tc_n_ok(row["Q"]), rid
    assert tuple(row["modes"]) == MODES and row["rectified"] in (0, 1) and row["reaches"], rid


def test_block_rows_reach_every_axis_value():
    rows = list(TS.BLOCK_ROWS.values())
    for mode in MODES:
        sel = [r for r in rows if mode in r["modes"]]
        assert {r["R"] for r in sel} == set(R_ALL), mode
        assert {r["S"] for r in sel} == set(S_ALL), mode
        assert {r["Ap"] for r in sel} == set(AP_ALL), mode
        assert {r["ks"] for r in sel} == set(KS_ALL), mode
        assert {(r["R"], r["ks"]) for r in sel} == set(itertools.product(R_ALL, KS_ALL)), mode
        assert {r["Ap"] for r in sel if r["ks"] == 3} == set(AP_ALL), mode
        assert {r["Ap"] for r in sel if r["R"] == 512} == set(AP_ALL), mode
        assert max(r["ks"] * r["R"] + r["Ap"] for r in sel) == 1792, mode
        assert {r["last"] for r in sel} == {False, True} and {r["init"] for r in sel} == {False, True}, mode
    # both tf32 backwards of a composed R = 64 forward are represented
    assert {r["tf32_bwd"] for r in rows if r["R"] == 64 and "tf32" in r["modes"]} == {"r64", "composed"}


def test_block_rows_reach_the_time_edges():
    rows = list(TS.BLOCK_ROWS.values())
    assert any(r["T"] == 1 for r in rows)
    assert any(r["T"] % 64 == 63 for r in rows) and any(r["T"] % 64 == 1 and r["T"] > 64 for r in rows)
    # an odd number of 64-row tiles over the batch: the last CTA of a two-tile pair (gemm_nt_tc.cu:650) is half empty
    assert any((r["B"] * -(-r["T"] // 64)) % 2 == 1 and r["B"] * -(-r["T"] // 64) > 1 for r in rows)
    assert any(r["d"] >= r["T"] for r in rows)
    # three utterances whose 64-row tiles straddle no boundary at a multiple of 64: tiles span batch rows
    assert any(r["B"] == 3 and r["T"] % 64 != 0 and r["T"] > 64 for r in rows)


def test_post_rows_reach_their_edges():
    rows = list(TS.POST_ROWS.values())
    assert {32, 96, 160, 224, 256, 512} <= {r["S"] for r in rows}
    assert {32, 160, 256, 512} <= {r["Q"] for r in rows}
    assert {r["rectified"] for r in rows} == {0, 1}
    assert any(post_split(r["S"]) for r in rows)
    # Q = 512: the N = 512 two-block plain GEMM, and a 4-M-block dWp2
    v = post_variants(256, 512, 0, "tf32")
    assert gemm("post2", "tf32", 512) == ("gemm", "post2", "tf32", 256, "plain", 2, "none", 1) and gemm(
        "post2", "tf32", 512) in v
    assert any(w[0] == "wgrad" and w[1] == "dWp2" and w[3] == 4 for w in v)
    # Ap / S of 160 and 224: nB = 1 with n_split 5 and 7
    for N, n_split in ((160, 5), (224, 7)):
        w = wgrad_concat("x", "tf32", N, False, 128, N, False)
        assert (w[5], w[7]) == (1, n_split)


# ------------------------------------------------------------------------------------------------------------------
# whole coverage: the library's predicate and the launch variants over the grid
# ------------------------------------------------------------------------------------------------------------------
def test_library_predicate_is_composed_tc_supported_over_the_grid():
    lib = _lib.load()
    sup = lib.wnb_resblock_fwd_supported
    n = {"fused": 0, "composed": 0}
    for R, S, Ap, ks in _block_grid():
        want = composed_tc_supported(R, S, Ap, ks)
        assert sup(R, S, Ap, ks, _lib.MATH_BF16) == (2 if want else 0), (R, S, Ap, ks)
        tf = sup(R, S, Ap, ks, _lib.MATH_TF32)
        assert tf == (1 if fused_fwd(R, S, Ap, ks) else 2 if want else 0), (R, S, Ap, ks)
        n["fused" if tf == 1 else "composed"] += tf > 0
    # the fused kernel takes R 64, ks 2, Ap 32 at every S that is a multiple of 64 (16 in the grid, 5 of them composed
    # shapes as well); the composed path the other 1 075 of its 1 080 shapes
    assert n == {"fused": 16, "composed": 1075}
    assert sum(composed_tc_supported(*s) for s in _block_grid()) == 1080
    assert sum(fused_fwd(*s) and composed_tc_supported(*s) for s in _block_grid()) == 5


def test_block_rows_reach_every_launch_variant_of_the_grid():
    want = set()
    for R, S, Ap, ks in _block_grid():
        for mode in row_modes(R, S, Ap, ks):
            for last in (False, True):
                want |= block_variants(R, S, Ap, ks, last, mode)
    got = set()
    for row in TS.BLOCK_ROWS.values():
        for mode in row["modes"]:
            got |= block_variants(*_shape(row), row["last"], mode)
    assert got <= want
    missing = sorted(want - got, key=repr)
    assert not missing, "%d launch variants no row reaches, e.g. %s" % (len(missing), missing[:8])
    # the issue's named gaps are among them
    assert gemm("gate_fwd", "tf32", 256, "gate", launches=2) in want                  # R = 256: two gate launches
    assert wgrad_concat("dW1_aux", "bf16", 512, False, 512, 224, False)[5:8] == (1, 0, 7)


def test_post_rows_reach_every_launch_variant_of_the_grid():
    want = set()
    for S, Q in itertools.product(GRID_RS, GRID_Q):
        if nt_tc_n_ok(S) and nt_tc_n_ok(Q):
            for mode in MODES:
                for rect in (0, 1):
                    want |= post_variants(S, Q, rect, mode)
    got = set()
    for row in TS.POST_ROWS.values():
        for mode in row["modes"]:
            got |= post_variants(row["S"], row["Q"], row["rectified"], mode)
    assert got <= want
    missing = sorted(want - got, key=repr)
    assert not missing, "%d launch variants no post row reaches, e.g. %s" % (len(missing), missing[:8])


def test_bf16_supported_agrees_with_the_library():
    from pytorchwavenetvocoder_b200.nets.wavenet import bf16_supported
    lib = _lib.load()
    n = 0
    for R, S, Ap, ks in _block_grid():
        blk = lib.wnb_resblock_fwd_supported(R, S, Ap, ks, _lib.MATH_BF16) == 2
        for Q in GRID_Q:
            lib_ok = blk and nt_tc_n_ok(S) and nt_tc_n_ok(Q)
            # the model pads n_aux up to a multiple of 32: n_aux = Ap - 5 pads to Ap
            assert bf16_supported((Q, Ap - 5, R, S, 4, 1, ks, 0)) == lib_ok, (Q, Ap, R, S, ks)
            n += lib_ok
    assert n == 1080 * 9
