# -*- coding: utf-8 -*-
"""CPU tier: the stack shape table (tests/stack_shapes.py) reaches the whole coverage of the deferred-skip stack and of
the fused R = 64 per-block path, from the library's coverage queries and from a restatement of their dispatch.

* over L in 1..80 and S in 32..2 048 the library's ``wnb_stack_supported`` is exactly ``stack_supported`` and
  ``wnb_resblock_fwd_supported`` exactly ``resblock_fwd_skip_supported`` / ``composed_tc_supported``;
* every stack row is a stack shape and every fused row a fused-forward, R = 64 gate-GEMM-backward shape;
* the launch variants of the stack rows are exactly those of every supported (L, S) with the aux gradient on and off,
  and the launch variants of the fused rows exactly those of every fused S with ``last``, ``init`` and dhaux both ways;
* the rows reach the time and dilation edges their docstring names.

A launch variant is what one launch instantiates or how the host splits its work: for the stack, the forward block
kernel's residual output and tile direction, the N and column blocks of the skip and dZ_all GEMMs (and whether dZ_all
is one block), the chain kernel's template (dhaux on or off), residual and tile direction, the form of the dx_0 launch,
and of the weight-gradient list the dWskip (M-block count, last-block rows, nB, M = 64 form) and the number of
``kMaxProb`` launches; for the fused path, the forward's residual chunk, skip init and whether its W2 chunk count is a
multiple of the ring depth, the dz / dX forms and each dW2 launch's (M-blocks, two-operand block, M = 64 form).  A new
instantiation or split that no row reaches makes the set equality fail."""
import itertools

import pytest

from pytorchwavenetvocoder_b200 import _lib
from tests import stack_shapes as SS

R, AP, KS = 64, 32, 2
GRID_L = range(1, 81)
GRID_S = range(32, 2049, 32)
STACK_S = (32, 64, 96, 128, 160, 192, 224, 256, 512)


# ------------------------------------------------------------------------------------------------------------------
# the dispatch, restated (csrc/stack.cu, csrc/stack_bwd_chain.cu, csrc/wgrad_tc.cu, csrc/resblock_z.cu,
# csrc/resblock_simt.cu, csrc/gemm_nt_tc.cu)
# ------------------------------------------------------------------------------------------------------------------
def fwd_z_supported(R_, Ap, ks):
    """resblock_z.cu:465 resblock_fwd_z_supported"""
    return R_ == 64 and ks == 2 and Ap == 32


def stack_supported(R_, S, Ap, ks, L):
    """stack.cu:42-47 stack_supported"""
    return fwd_z_supported(R_, Ap, ks) and 1 <= L <= 64 and S % 32 == 0 and S >= 32 and (S <= 256 or S == 512)


def fused_fwd(R_, S, Ap, ks):
    """resblock_z.cu:496-498 resblock_fwd_skip_supported"""
    return R_ == 64 and ks == 2 and Ap == 32 and S >= 64 and S % 64 == 0


def tc_fused_shape(R_, S, Ap, ks):
    """resblock_simt.cu:719 tc_fused_shape (tf32): the R = 64 gate-GEMM backward"""
    return R_ == 64 and ks == 2 and Ap == 32 and S % 32 == 0


def composed_tc_supported(R_, S, Ap, ks):
    """resblock_simt.cu:574-576 composed_tc_supported"""
    def n_ok(N):
        return N % 32 == 0 and N >= 32 and (N <= 256 or N == 512)
    return R_ % 64 == 0 and n_ok(R_) and n_ok(S) and Ap % 32 == 0 and Ap <= 256 and 1 <= ks <= 3


def pick_block(total, cands=(256, 192, 128, 64, 32)):
    """stack.cu:27-31 pick_block, with the dZ_all candidates of stack.cu:150"""
    return next((c for c in cands if total % c == 0), 0)


def gemm_nblk(N):
    """gemm_nt_tc.cu:547-554: N = 512 runs as two column blocks of 256"""
    return (256, 2) if N == 512 else (N, 1)


def dwskip_nb(L):
    """stack.cu:238-243: the largest column group count c <= 7 that divides L*R/32 into at most 128 groups"""
    groups = L * R // 32
    return next(c for c in range(7, 0, -1) if groups % c == 0 and groups // c <= 128)


def wgrad_nA(m_valid, nB, ones):
    """wgrad_tc.cu:521, :544 pr.nA: the M = 64 form (2 A sub-tiles) for m_valid <= 64 and N = 32 (nB + ones) <= 128"""
    return 2 if (m_valid <= 64 and 32 * (nB + ones) <= 128) else 4


K_MAX_PROB = 160   # wgrad_tc.cu:49 kMaxProb: problems per launch (the list is cut at :607-608)


def stack_problems(L, S):
    """the problem list of wnb_stack_bwd's one wgrad_tc_multi call (stack.cu:216-257, wgrad_tc.cu:538-592): L dW1
    segments, L - 1 dW2res segments and the dWskip M-blocks x column groups; returns (count, dWskip variants)"""
    nB = dwskip_nb(L)
    groups = L * R // 32
    nmb = (S + 127) // 128                                   # stack.cu:239
    m_last = S - 128 * (nmb - 1)                             # stack.cu:251 m_valid of the last M-block
    dws = {("dWskip", nmb, m_last, nB, wgrad_nA(m_last, nB, 1))}
    count = L + (L - 1) + nmb * (groups // nB)
    return count, dws


def stack_variants(L, S, aux, alt_dir=True):
    """the launches of wnb_stack_fwd (stack.cu:81-108) and wnb_stack_bwd (stack.cu:127-258)"""
    assert stack_supported(R, S, AP, KS, L)
    rev = (lambda k: k & 1) if alt_dir else (lambda k: 0)    # stack.cu:37-40 alternate_dir
    v = set()
    for l in range(L):   # stack.cu:96-105: xout unless last, block l reversed if odd
        v.add(("fwd_z", l + 1 < L, rev(l)))
    v.add(("skip_gemm",) + gemm_nblk(S))                     # stack.cu:70-79
    ldz = L * R
    nb = pick_block(ldz)                                     # stack.cu:149-159
    v.add(("dzall", nb, ldz // nb == 1))
    v.add(("gate_bwd_last", rev(0)))                         # stack.cu:168-182: N 128 gate backward, no z
    for l in range(L - 1, 0, -1):                            # stack.cu:184-191
        # stack_bwd_chain.cu:369, :390: template AUX = dhaux given; :382 has_res = dx_{l+1} given; direction of
        # launch L - l
        v.add(("chain", aux, l + 1 < L, rev(L - l)))
    # stack.cu:192-211: dx_0 with dhaux N = R + Ap and a split output, without N = R; residual = dx_1 unless L = 1
    v.add(("dx0", aux, L > 1, rev(L)))
    n, dws = stack_problems(L, S)
    v |= dws
    v.add(("wgrad_launches", -(-n // K_MAX_PROB)))
    return v


R64_KSLOT = 2   # resblock_z.cu:243 tcs::kSNSlot: the W2 chunk ring of the fused forward


def fused_variants(S, last, init, dhaux):
    """resblock_fwd_skip (resblock_z.cu:501-527, chunks :268) and the R = 64 gate-GEMM backward of wnb_resblock_bwd
    (resblock_simt.cu:782-871)"""
    assert fused_fwd(R, S, AP, KS) and tc_fused_shape(R, S, AP, KS)
    nchunks = (0 if last else 1) + S // 64
    v = {("fwd_skip", last, init, nchunks % R64_KSLOT == 0)}
    dout = not last
    v.add(("r64_dz", dout))                                   # :786-792
    v.add(("r64_gate",))                                      # :794-796
    v.add(("r64_dx", dhaux, dout))                            # :807-817
    v.add(("r64_dW1",))                                       # :841-845
    # :848-869: M-blocks of 128 rows from row_first, a launch every 5 blocks and after the last
    v |= r64_dw2_launches(S, dout)
    return v


def r64_dw2_launches(S, dout):
    """resblock_simt.cu:849-869: per wgrad_tc_blocks launch (M-blocks, a two-operand [dout | dskip] block, an M = 64
    problem)"""
    M = R + S
    out, blk = set(), []
    for r0 in range(0 if dout else R, M, 128):
        m_valid = min(128, M - r0)
        blk.append((r0 == 0, wgrad_nA(m_valid, 2, 1) == 2))
        if len(blk) == 5 or r0 + 128 >= M:
            out.add(("r64_dW2", len(blk), any(b[0] for b in blk), any(b[1] for b in blk)))
            blk = []
    assert not blk
    return out


# ------------------------------------------------------------------------------------------------------------------
# the rows
# ------------------------------------------------------------------------------------------------------------------
def _stack_row_variants(row, alt_dir=True):
    return stack_variants(row["L"], row["S"], row["aux"], alt_dir)


@pytest.mark.parametrize("rid", list(SS.STACK_ROWS))
def test_stack_row_takes_the_stack(rid):
    row = SS.STACK_ROWS[rid]
    lib = _lib.load()
    L, S = row["L"], row["S"]
    assert lib.wnb_stack_supported(R, S, AP, KS, L, _lib.MATH_TF32) == 1, rid
    assert stack_supported(R, S, AP, KS, L), rid
    assert len(row["dilations"]) == L and min(row["dilations"]) >= 1, rid
    assert row["B"] >= 1 and (row["T"] is None or row["T"] >= 1), rid
    assert row["relu"] in (0, 1) and row["aux"] in (False, True) and row["reaches"], rid


@pytest.mark.parametrize("rid", list(SS.FUSED_ROWS))
def test_fused_row_takes_the_fused_path(rid):
    row = SS.FUSED_ROWS[rid]
    lib = _lib.load()
    S = row["S"]
    assert lib.wnb_resblock_fwd_supported(R, S, AP, KS, _lib.MATH_TF32) == 1, rid     # the fused forward
    assert fused_fwd(R, S, AP, KS) and tc_fused_shape(R, S, AP, KS), rid              # and the R = 64 backward
    assert row["B"] >= 1 and row["T"] >= 1 and row["d"] >= 1, rid
    assert row["last"] in (False, True) and row["init"] in (False, True) and row["aux"] in (False, True), rid
    assert row["reaches"], rid


def test_the_six_stage_cases_are_kept():
    """the cases of test_gpu_tc_stages.test_stack_stages, unchanged (case d's T is derived from the SM count)"""
    want = {"a": (1, 32, 1, 1, [1]), "b": (3, 96, 2, 95, [1, 64, 200]), "c": (5, 512, 3, 1040, [1, 2, 4, 8, 16]),
            "d": (22, 256, 1, None, [2 ** (i % 10) for i in range(22)]),
            "e": (30, 512, 2, 8300, [2 ** i for i in range(10)] * 3),
            "f": (64, 128, 1, 200, [(37 * i) % 300 + 1 for i in range(64)])}
    for case, (L, S, B, T, dil) in want.items():
        row = SS.STACK_ROWS["case_" + case]
        assert (row["L"], row["S"], row["B"], row["T"], row["dilations"], row["aux"]) == (L, S, B, T, dil, True), case
    assert set(SS.STAGE_CASES) == set(want)


def test_stack_rows_reach_every_axis_value():
    rows = list(SS.STACK_ROWS.values())
    assert {r["S"] for r in rows} == set(STACK_S)
    # every skip width with every dWskip nB the stack can take (2 L / 32 groups: nB 3 never, 1 never)
    nbs = {dwskip_nb(L) for L in range(1, 65)}
    assert nbs == {2, 4, 5, 6, 7}
    assert {(r["S"], dwskip_nb(r["L"])) for r in rows} >= set(itertools.product(STACK_S, nbs))
    # ... at the smallest depth that has it (L = 1, 2, 3, 5, 7), and not only inside a deep case
    small = (1, 2, 3, 5, 7)
    assert {dwskip_nb(L) for L in small} == nbs
    grid_rows = [r for rid, r in SS.STACK_ROWS.items() if not rid.startswith("case_")]
    assert {(r["S"], r["L"]) for r in grid_rows if r["L"] in small} == set(itertools.product(STACK_S, small))
    assert {r["relu"] for r in rows} == {0, 1} and {r["aux"] for r in rows} == {False, True}
    # dx_0 meets L = 1, even L and odd L > 1 with the aux gradient on and off
    parity = lambda L: "one" if L == 1 else ("even" if L % 2 == 0 else "odd")   # noqa: E731
    assert {(r["aux"], parity(r["L"])) for r in rows} == set(itertools.product((False, True), ("one", "even", "odd")))
    # the longest weight-gradient list of the coverage: three launches (L = 59 or 61 at S = 512)
    assert {L for L in range(1, 65) if -(-stack_problems(L, 512)[0] // K_MAX_PROB) == 3} == {59, 61}
    assert any(r["L"] in (59, 61) and r["S"] == 512 for r in rows)


def test_stack_rows_reach_the_time_edges():
    rows = [r for r in SS.STACK_ROWS.values() if r["T"] is not None]
    tiles = lambda r: r["B"] * -(-r["T"] // 64)   # noqa: E731
    assert any(r["T"] == 1 for r in rows)
    assert any(r["T"] < 64 and r["L"] >= 2 for r in rows)                    # one tile per utterance in every launch
    assert any(r["T"] % 64 == 63 for r in rows) and any(r["T"] % 64 == 1 and r["T"] > 64 for r in rows)
    # odd tile counts: the last pair of the chain / gemm_nt_tc half empty (B = 1), pairs spanning utterances (B = 3)
    for B in (1, 3):
        assert any(r["B"] == B and tiles(r) % 2 == 1 and tiles(r) > 1 for r in rows), B
    assert any(r["L"] >= 2 and max(r["dilations"]) >= r["T"] > 1 for r in rows)
    # the chain kernel reads dpre_l at t + d_l and x_{l-1} at t - d_{l-1}: neighbouring dilations far apart
    assert any(any(abs(a - b) >= 256 for a, b in zip(r["dilations"], r["dilations"][1:])) for r in rows)


def test_fused_rows_reach_every_axis_value():
    rows = list(SS.FUSED_ROWS.values())
    assert {128, 256, 320, 384, 448, 576, 640, 1024} <= {r["S"] for r in rows}
    assert {r["last"] for r in rows} == {False, True} and {r["init"] for r in rows} == {False, True}
    assert {(r["last"], r["aux"]) for r in rows} == set(itertools.product((False, True), (False, True)))
    # the dW2 loop's last launch flush when R + S - row_first is a multiple of 128 and when it is not; R + S > 640
    # (more than 5 M-blocks) with and without dout
    assert {r["last"] for r in rows if R + r["S"] > 640} == {False, True}
    # W2 chunk counts that are not a multiple of the forward's ring depth
    assert any(((0 if r["last"] else 1) + r["S"] // 64) % R64_KSLOT != 0 for r in rows)
    assert any(((0 if r["last"] else 1) + r["S"] // 64) % R64_KSLOT == 0 for r in rows)
    # widths only the fused path trains (the stack takes S <= 256 and 512)
    assert {r["S"] for r in rows if r["S"] not in STACK_S} >= {320, 384, 448, 576, 640, 1024}


def test_fused_rows_reach_the_time_edges():
    rows = list(SS.FUSED_ROWS.values())
    tiles = lambda r: r["B"] * -(-r["T"] // 64)   # noqa: E731
    assert any(r["T"] == 1 for r in rows)
    assert any(r["T"] % 64 == 63 for r in rows) and any(r["T"] % 64 == 1 and r["T"] > 64 for r in rows)
    for B in (1, 3):
        assert any(r["B"] == B and tiles(r) % 2 == 1 and tiles(r) > 1 for r in rows), B
    assert any(r["d"] >= r["T"] > 1 for r in rows)


# ------------------------------------------------------------------------------------------------------------------
# whole coverage: the library's predicates and the launch variants over the grid
# ------------------------------------------------------------------------------------------------------------------
def test_library_predicates_over_the_grid():
    lib = _lib.load()
    n_stack = n_fused = 0
    for R_, Ap, ks in itertools.product((64, 128), (32, 64), (1, 2, 3)):
        for S in GRID_S:
            for L in GRID_L:
                want = stack_supported(R_, S, Ap, ks, L)
                assert lib.wnb_stack_supported(R_, S, Ap, ks, L, _lib.MATH_TF32) == int(want), (R_, S, Ap, ks, L)
                n_stack += want
            assert lib.wnb_stack_supported(R_, S, Ap, ks, 8, _lib.MATH_BF16) == 0, (R_, S, Ap, ks)
            tf = lib.wnb_resblock_fwd_supported(R_, S, Ap, ks, _lib.MATH_TF32)
            assert tf == (1 if fused_fwd(R_, S, Ap, ks) else 2 if composed_tc_supported(R_, S, Ap, ks) else 0), \
                (R_, S, Ap, ks)
            n_fused += tf == 1
    assert n_stack == 9 * 64 and n_fused == 2048 // 64


def _stack_grid():
    for L, S in itertools.product(GRID_L, GRID_S):
        if stack_supported(R, S, AP, KS, L):
            yield L, S


def _grid_stack_variants():
    want = set()
    for L, S in _stack_grid():
        for aux in (False, True):
            want |= stack_variants(L, S, aux)
    return want


def test_stack_rows_reach_every_launch_variant_of_the_grid():
    want = _grid_stack_variants()
    got = set()
    for row in SS.STACK_ROWS.values():
        got |= _stack_row_variants(row)
    assert got <= want
    missing = sorted(want - got, key=repr)
    assert not missing, "%d launch variants no stack row reaches, e.g. %s" % (len(missing), missing[:8])
    assert len(want) == SS.STACK_VARIANTS, len(want)
    # the six stage cases alone leave most of them unreached
    six = set()
    for case in SS.STAGE_CASES:
        six |= _stack_row_variants(SS.STACK_ROWS["case_" + case])
    assert len(six) < len(want) // 2


def test_stack_variants_name_the_issue_s_gaps():
    want = _grid_stack_variants()
    for N in (64, 160, 192, 224):
        assert ("skip_gemm", N, 1) in want
    assert ("dzall", 128, True) in want and ("dzall", 256, True) in want
    assert any(v[0] == "dWskip" and v[3] == 7 for v in want)
    # the M = 64 dWskip form after a full M-block: S = 160 / 192 with nB = 2 (L = 1)
    assert ("dWskip", 2, 32, 2, 2) in want and ("dWskip", 2, 64, 2, 2) in want
    assert ("chain", False, False, 1) in want and ("dx0", False, True, 0) in want
    assert ("wgrad_launches", 3) in want
    # WNB_ALT_DIR=0 leaves only front-to-back launches
    assert all(v[-1] == 0 for v in stack_variants(7, 256, True, alt_dir=False) if v[0] in ("fwd_z", "chain", "dx0"))


def _fused_grid():
    for S in GRID_S:
        if fused_fwd(R, S, AP, KS):
            yield S


def test_fused_rows_reach_every_launch_variant_of_the_grid():
    want = set()
    for S in _fused_grid():
        for last, init, dh in itertools.product((False, True), repeat=3):
            want |= fused_variants(S, last, init, dh)
    got = set()
    for row in SS.FUSED_ROWS.values():
        got |= fused_variants(row["S"], row["last"], row["init"], row["aux"])
    assert got <= want
    missing = sorted(want - got, key=repr)
    assert not missing, "%d launch variants no fused row reaches, e.g. %s" % (len(missing), missing[:8])
    assert len(want) == SS.FUSED_VARIANTS, len(want)


def test_r64_dw2_flush_rule():
    """the dW2 loop launches after every 5th M-block and after the last one, whether or not that one is full"""
    assert r64_dw2_launches(192, True) == {("r64_dW2", 2, True, False)}       # 256 rows: the last block is full
    assert r64_dw2_launches(128, True) == {("r64_dW2", 2, True, True)}        # 192 rows: the last block has 64
    assert r64_dw2_launches(1024, False) == {("r64_dW2", 5, False, False), ("r64_dW2", 3, False, False)}
    assert r64_dw2_launches(640, True) == {("r64_dW2", 5, True, False), ("r64_dW2", 1, False, True)}
