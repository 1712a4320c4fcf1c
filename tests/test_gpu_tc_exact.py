# -*- coding: utf-8 -*-
"""GPU tier: the linear tensor-core entry points with EXACT arithmetic.

Inputs are small integers, chosen so that every operand entering a multiply has at most 11 significant bits (exact in
tf32 under either conversion rule) and every partial sum stays below 2^24 (exact in fp32 in any summation order).  The
kernels' results must then equal the float64 result bit for bit: a single missing, duplicated or shifted term -- a
dropped partial time tile, a CTA that skips or repeats a tile, two column groups swapped, = where += belongs -- fails.

The first test measures how the tensor cores read an fp32 operand whose low mantissa bits are set (the kernels issue
no cvt: wgmma reads the fp32 bit pattern as tf32) and pins the rule tests/tc_reference.py assumes.
"""
import pytest
import torch

from tests import tc_reference as ref

pytestmark = pytest.mark.gpu

SMALL_T = (1, 31, 33, 63, 65)


def _lib():
    from pytorchwavenetvocoder_b200 import _lib as L
    return L, L.load()


def _ints(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).to(torch.float32)


def _skip_gemm(zall, wskip, bskip, relu):
    L, lib = _lib()
    B, T, K = zall.shape
    S = wskip.shape[0]
    out = torch.full((B, T, S), float("nan"), device="cuda")
    L.check(lib.wnb_skip_gemm(L.ptr(zall), L.ptr(wskip), L.ptr(bskip), L.ptr(out), B, T, K, S, relu, L.stream()),
            "skip_gemm")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("side", ["activation", "weight"])
def test_tf32_conversion_rule(side, sign):
    """One nonzero product v * 1.0 with v = +-(1 + 2^-11 + 2^-12): its bits below the tf32 mantissa are 0b11, so
    truncation gives +-1 and round-to-nearest gives +-(1 + 2^-10)."""
    K = S = 32
    v = sign * (1.0 + 2.0 ** -11 + 2.0 ** -12)
    zall = torch.zeros(1, 1, K, device="cuda")
    wskip = torch.zeros(S, K, device="cuda")
    k0, n0 = 13, 21
    zall[0, 0, k0] = v if side == "activation" else 1.0
    wskip[n0, k0] = 1.0 if side == "activation" else v
    out = _skip_gemm(zall, wskip, None, 0)
    got = float(out[0, 0, n0])
    found = {sign * 1.0: "truncate", sign * (1.0 + 2.0 ** -10): "round"}.get(got)
    print("tf32 operand conversion (%s, sign %+d): %.10f -> %s" % (side, sign, got, found))
    assert found is not None, got
    assert found == ref.TF32_RULE, (found, ref.TF32_RULE)
    assert float(ref.to_tf32(torch.tensor([v]))[0]) == got
    others = torch.cat([out[0, 0, :n0], out[0, 0, n0 + 1:]])
    assert torch.equal(others, torch.zeros_like(others))


# S, K pairs: every N instantiation the skip GEMM uses (S = 512: two 256-column blocks) and K from one to 128 chunks
_SK = [(32, 32), (96, 4096), (224, 160), (256, 1920), (512, 640)]
_SHAPES = [(2, t) for t in SMALL_T] + [(2, 8300)]


@pytest.mark.parametrize("B,T", _SHAPES)
@pytest.mark.parametrize("S,K", _SK)
@pytest.mark.parametrize("relu", [0, 1])
def test_skip_gemm_exact(S, K, B, T, relu):
    g = torch.Generator(device="cuda").manual_seed(S * 7 + K + T + relu)
    zall = _ints(g, (B, T, K), -7, 7)
    wskip = _ints(g, (S, K), -7, 7)
    bskip = _ints(g, (S,), -50, 50)
    got = _skip_gemm(zall, wskip, bskip, relu)
    want = zall.double() @ wskip.double().t() + bskip.double()
    if relu:
        want = want.clamp_min(0)
    if not torch.equal(got, want.float()):
        r, i = ref.worst(got, want, torch.zeros_like(want))
        raise AssertionError("skip_gemm S=%d K=%d: first wrong element %s" % (S, K, ref.locate(got.shape, i)))


def _post_fwd(skip, wp1, bp1, wp2, bp2, rectified):
    L, lib = _lib()
    B, T, S = skip.shape
    Q = wp2.shape[0]
    r1 = torch.full((B, T, S), float("nan"), device="cuda")
    logits = torch.full((B, T, Q), float("nan"), device="cuda")
    L.check(lib.wnb_post_fwd(L.ptr(skip), L.ptr(wp1), L.ptr(bp1), L.ptr(wp2), L.ptr(bp2), L.ptr(r1), L.ptr(logits),
                             B, T, S, Q, L.MATH_TF32, rectified, L.stream()), "post_fwd")
    torch.cuda.synchronize()
    return r1, logits


@pytest.mark.parametrize("B,T", _SHAPES)
@pytest.mark.parametrize("S", [512, 256])
def test_post_fwd_exact(S, B, T):
    """S = 512 takes the two-column-block split of the first GEMM.  skip in {-1..2} (rectified in place by the call),
    wp1 in {-1, 0, 1}: |h1| <= 2 S + 3 < 2^11, so r1 is an exact tf32 operand of the second GEMM."""
    Q = 256
    g = torch.Generator(device="cuda").manual_seed(S + T)
    skip = _ints(g, (B, T, S), -1, 2)
    wp1, bp1 = _ints(g, (S, S), -1, 1), _ints(g, (S,), -3, 3)
    wp2, bp2 = _ints(g, (Q, S), -3, 3), _ints(g, (Q,), -9, 9)
    sk0 = skip.clone()
    r1, logits = _post_fwd(skip, wp1, bp1, wp2, bp2, 0)
    sr = sk0.double().clamp_min(0)
    assert torch.equal(skip, sr.float())             # rectified in place
    h1 = (sr @ wp1.double().t() + bp1.double()).clamp_min(0)
    assert h1.abs().max().item() < 2048
    assert torch.equal(r1, h1.float()), ref.locate(r1.shape, ref.worst(r1, h1, torch.zeros_like(h1))[1])
    want = h1 @ wp2.double().t() + bp2.double()
    assert torch.equal(logits, want.float()), ref.locate(logits.shape, ref.worst(logits, want, torch.zeros_like(want))[1])


@pytest.mark.parametrize("B,T", [(2, t) for t in SMALL_T] + [(3, 700)])
@pytest.mark.parametrize("S", [512, 256])
def test_post_bwd_exact(S, B, T):
    """Mask epilogues (r1 > 0, skip > 0) and the weight gradients through wgrad_tc_concat: dWp1 with S/128 M-blocks,
    dWp2 with Q/128, column groups across CTAs (n_split) and the all-ones bias column.  The gradient buffers start at
    nonzero values, which must be accumulated into.  |dh1| <= 2 * 3 * Q < 2^11 and B*T*max|dh1*skip| < 2^24."""
    L, lib = _lib()
    Q = 256
    g = torch.Generator(device="cuda").manual_seed(3 * S + T)
    skip = _ints(g, (B, T, S), -2, 2).clamp_min(0)          # what the tf32 forward leaves: rectified
    r1 = _ints(g, (B, T, S), -3, 3).clamp_min(0)
    dlogits = _ints(g, (B, T, Q), -2, 2)
    wp1, wp2 = _ints(g, (S, S), -1, 1), _ints(g, (Q, S), -3, 3)
    wp1t, wp2t = wp1.t().contiguous(), wp2.t().contiguous()
    init = {k: _ints(g, sh, -5, 5) for k, sh in (("dwp1", (S, S)), ("dbp1", (S,)), ("dwp2", (Q, S)), ("dbp2", (Q,)))}
    out = {k: v.clone() for k, v in init.items()}
    dskip = torch.full((B, T, S), float("nan"), device="cuda")
    ws = torch.full((B, T, S), float("nan"), device="cuda")
    L.check(lib.wnb_post_bwd(L.ptr(skip), L.ptr(r1), L.ptr(dlogits), L.ptr(wp1t), L.ptr(wp2t), L.ptr(dskip),
                             L.ptr(out["dwp1"]), L.ptr(out["dbp1"]), L.ptr(out["dwp2"]), L.ptr(out["dbp2"]), L.ptr(ws),
                             B, T, S, Q, L.MATH_TF32, L.stream()), "post_bwd")
    torch.cuda.synchronize()
    D = lambda t: t.double().reshape(-1, t.shape[-1])   # noqa: E731
    dh1 = (dlogits.double() @ wp2.double()) * (r1 > 0)
    assert dh1.abs().max().item() < 2048
    dsk = (dh1 @ wp1.double()) * (skip > 0)
    want = {"dwp2": init["dwp2"].double() + D(dlogits).t() @ D(r1), "dbp2": init["dbp2"].double() + D(dlogits).sum(0),
            "dwp1": init["dwp1"].double() + D(dh1).t() @ D(skip), "dbp1": init["dbp1"].double() + D(dh1).sum(0)}
    assert torch.equal(ws, dh1.float()), ("dh1", ref.locate(ws.shape, ref.worst(ws, dh1, torch.zeros_like(dh1))[1]))
    assert torch.equal(dskip, dsk.float()), ("dskip", ref.locate(dskip.shape, ref.worst(dskip, dsk, 0 * dsk)[1]))
    for k, w in want.items():
        assert w.abs().max().item() < 2 ** 24
        assert torch.equal(out[k], w.float()), (k, ref.locate(out[k].shape, ref.worst(out[k], w, 0 * w)[1]))
