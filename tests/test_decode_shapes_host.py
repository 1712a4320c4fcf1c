# -*- coding: utf-8 -*-
"""CPU tier: every row of the decode shape table (tests/decode_shapes.py) reaches the branch it claims, from the
library's coverage queries and from restatements of the launch rules:

* ``wnb_decode_stream_supported`` and ``wnb_decode_warp_supported`` send the row where the table says;
* streaming rows: NU and the ring slots (``stream_plan``, restated in test_decode_stream_pool_host.py), and the parts
  and rows per chunk of every width (``parts_for``, ``rows_per_chunk``);
* direct rows: NU after ``decode_smem_floats``' halving and the widths that take ``gemv_partial``'s wide-output loop;
* the direct carve-up puts ``partial`` at a multiple of 4 floats on a grid of shapes that includes every row."""
import itertools

import pytest

from pytorchwavenetvocoder_b200 import _lib
from tests import decode_shapes as T
from tests.test_decode_stream_pool_host import _stream_plan

SMS = T.SMS_H100


def parts_for(O):
    """decode_stream.cu parts_for (and decode.cu gemv_partial's parts below 256 lanes)"""
    lanes = O // 4
    return 1 if lanes >= 256 else 256 // lanes


def rows_per_chunk(O, parts):
    """decode_stream.cu rows_per_chunk"""
    r = 32 * 1024 // (O * 4)
    if r > parts:
        r = r // parts * parts
    return max(r, 1)


def stream_widths(Q, R, S):
    return {"O1": T.round4(2 * R), "Or": T.round4(R), "Os": T.round4(S), "Sp": T.round4(S), "Qp": T.round4(Q)}


def direct_widths(Q, R, S):
    return {"O1": T.round4(2 * R), "O2": T.round4(R + S), "O2_warmup": T.round4(R), "Sp": T.round4(S),
            "Qp": T.round4(Q)}


def sampler_lanes(Q):
    """classes per sampler lane: chunk = ceil(Q / 32), lane l owns [l chunk, min((l + 1) chunk, Q))"""
    c = (Q + 31) // 32
    return [max(0, min((l + 1) * c, Q) - l * c) for l in range(32)]


def _facts(row):
    Q, Ap, R, S, ks, L = T.kernel_dims(row)
    out = {"Ap": Ap, "L": L, "stream": [], "direct": []}
    for bfn in row["batches"]:
        B = bfn(SMS)
        nu0 = T.first_nu(B, SMS)
        out["stream"].append(_stream_plan(Q, Ap, R, S, ks, L, nu0))
        out["direct"].append(T.direct_plan(Q, Ap, R, S, ks, L, nu0))
    sw = stream_widths(Q, R, S)
    out["parts"] = {k: parts_for(v) for k, v in sw.items()}
    out["rpc"] = {k: rows_per_chunk(v, parts_for(v)) for k, v in sw.items()}
    out["wide"] = sorted(k for k, v in direct_widths(Q, R, S).items() if v // 4 > 256)
    out["lanes"] = sampler_lanes(Q)
    return out


@pytest.mark.parametrize("rid", list(T.ROWS))
def test_row_takes_the_decoder_it_claims(rid):
    row = T.ROWS[rid]
    lib = _lib.load()
    Q, Ap, R, S, ks, L = T.kernel_dims(row)
    f = _facts(row)
    assert len(T.dilations(row)) == row["shape"][4] * row["shape"][5], rid    # the model has one layer per dilation
    assert not lib.wnb_decode_warp_supported(Q, Ap, R, S, ks, L), rid
    assert bool(lib.wnb_decode_stream_supported(Q, Ap, R, S, ks, L)) == (row["rule"] == "stream"), rid
    if row["rule"] == "stream":
        assert all(p is not None for p in f["stream"]), (rid, f["stream"])
    elif row["rule"] == "direct":
        assert all(p is None for p in f["stream"]) and all(p is not None for p in f["direct"]), (rid, f)
    else:
        assert all(p is None for p in f["stream"] + f["direct"]), (rid, f)
    # every plan's NU must divide none of the batch sizes: the last CTA is partly empty
    for bfn, p in zip(row["batches"], f["stream"] if row["rule"] == "stream" else f["direct"]):
        if p is not None and p[0] > 1:
            assert bfn(SMS) % p[0] != 0, rid


def test_rows_reach_their_branches():
    """the claim of every row, from the restated launch rules"""
    F = {rid: _facts(row) for rid, row in T.ROWS.items()}
    # Q 1 024: Qp 256 lanes, parts 1, 32 classes per sampler lane
    assert F["q1024"]["parts"]["Qp"] == 1 and F["q1024"]["lanes"] == [32] * 32
    # Q 1 022: two padded columns, short last lane
    assert T.round4(1022) - 1022 == 2 and F["q1022"]["lanes"] == [32] * 31 + [30]
    # odd parts: 42 / 85 / 28, each leaving threads idle, K = R = 12 below the W2res parts; lanes with 1 class and none
    p = F["odd_parts"]["parts"]
    assert (p["O1"], p["Or"], p["Os"], p["Sp"], p["Qp"]) == (42, 85, 85, 85, 28)
    assert all(256 % (T.round4(w) // 4) != 0 for w in (24, 12, 36))
    assert 12 < p["Or"]
    assert F["odd_parts"]["lanes"] == [2] * 16 + [1] + [0] * 15
    assert [s[0] for s in F["odd_parts"]["stream"]] == [1, 2, 4]
    # widest: 256-lane O1 and Os (parts 1), NU 4 -> 2 at B > 2 SMs
    assert F["widest"]["parts"]["O1"] == F["widest"]["parts"]["Os"] == F["widest"]["parts"]["Sp"] == 1
    assert stream_widths(256, 512, 1024)["O1"] // 4 == 256
    assert [s[0] for s in F["widest"]["stream"]] == [1, 2]
    assert T.first_nu(T.ROWS["widest"]["batches"][1](SMS), SMS) == 4
    # the shared-memory edge: L 36 runs on two ring slots, L 37 is refused
    assert F["smem_edge"]["stream"] == [(1, 2)] and F["smem_edge"]["Ap"] == 96 and F["smem_edge"]["L"] == 36
    assert F["smem_edge_l37"]["L"] == 37 and F["smem_edge_l37"]["stream"] == [None]
    # ks 1, 4, 5
    assert T.ROWS["ks1"]["shape"][6] == 1
    for rid, ks in (("ks4", 4), ("ks5", 5)):
        d = T.dilations(T.ROWS[rid])
        assert T.ROWS[rid]["shape"][6] == ks and 1 in d and max(d) > T.ROWS[rid]["max_n"]
        assert any(v & (v - 1) for v in d)            # a dilation that is not a power of two
    # L 64: kMaxLayersS, a 1-lane Or, 256-lane Os
    assert F["l64"]["L"] == 64 and F["l64"]["parts"]["Or"] == 256 and F["l64"]["parts"]["Os"] == 1
    # direct: the wide-output loop
    assert F["r516"]["wide"] == ["O1"]
    assert F["s1028_q1028"]["wide"] == ["O2", "Qp", "Sp"]
    assert F["d1"]["wide"] == [] and F["odd_rs_q255"]["wide"] == []
    # direct: NU 4 -> 2
    assert T.first_nu(T.ROWS["direct_nu_halves"]["batches"][0](SMS), SMS) == 4
    assert F["direct_nu_halves"]["direct"][0][0] == 2
    assert [d[0] for d in F["d1"]["direct"]] == [1, 2]
    # neither: over 64 layers, over 227 KB at NU 1
    Q, Ap, R, S, ks, L = T.kernel_dims(T.ROWS["smem_over"])
    omax = max(T.round4(Q), 1024)
    assert 4 * (T.direct_partial_offset(1, Q, Ap, R, S, ks, L) + omax) > 227 * 1024 and L <= 64
    assert F["l65"]["L"] == 65


def test_misaligned_rows_need_the_rounding():
    """the rows that would have stored float4 at an 8-byte boundary before partial's offset was rounded up"""
    for rid, nu, mod in (("d1", 1, 2), ("odd_rs_q255", 1, 3), ("direct_nu_halves", 1, 2)):
        assert T.direct_scalar_floats(nu, *T.kernel_dims(T.ROWS[rid])) % 4 == mod, rid
    assert T.direct_scalar_floats(1, *T.kernel_dims(T.ROWS["d1"])) == 378
    # the issue's other examples: R = 30, S = 32, L = 1; Q = 255, R = S = 6, ks 3, L = 5
    assert T.direct_scalar_floats(1, 256, 32, 30, 32, 2, 1) % 4 == 2
    assert T.direct_scalar_floats(1, 255, 32, 6, 6, 3, 5) % 4 == 2


def test_partial_offset_is_16_byte_aligned_over_a_grid():
    """decode.cu decode_partial_offset: a multiple of 4 floats, at most 3 past the scalar regions, for every shape of a
    grid that includes every row of the table, at NU 1, 2 and 4"""
    shapes = set(T.kernel_dims(r) for r in T.ROWS.values())
    for Q, A, R, S, ks, L in itertools.product((2, 33, 255, 256, 1022, 1028), (1, 28, 80, 256), (1, 2, 3, 6, 7, 30, 254,
                                               516), (1, 8, 9, 32, 1028), (1, 2, 3, 4, 5), (1, 3, 5, 22, 37, 64)):
        shapes.add((Q, T.n_aux_pad(A), R, S, ks, L))
    n_mis = 0
    for dims in shapes:
        Q, Ap, R, S, ks, L = dims
        for nu in (1, 2, 4):
            # the kernel's pointer chain xcat, cur, zs, skipacc, h1, logit, hcol, qtap, then partial_pad
            walk = (nu * (ks * R + Ap) + nu * R + nu * R + nu * S + nu * S + nu * T.round4(Q) + nu * Ap
                    + nu * (ks - 1) * L * R)
            raw = T.direct_scalar_floats(nu, *dims)
            off = T.direct_partial_offset(nu, *dims)
            assert walk == raw, (dims, nu)
            assert off % 4 == 0 and 0 <= off - raw <= 3, (dims, nu)
            n_mis += raw % 4 != 0
    assert n_mis > 1000    # the grid holds many shapes the rounding moves
