# -*- coding: utf-8 -*-
"""GPU tier: every stage of the fp32 (SIMT, ``math_mode="fp32"``) path against float64, element by element.

The fp32 path (csrc/resblock_simt.cu over the FFMA main loop of csrc/gemm_simt.cuh) is the parity mode, and other tests
use it as their truth, so it is checked here with the element-wise bounds of tests/tc_reference.py for fp32 operands
(``cv=exact``: operands as given, every product exact in float64) and the SIMT gate functions (``gate_fn=GATE_LIBM``:
``1 / (1 + expf(-a))`` and ``tanhf``, each within 2 ulp).  Teacher forcing: each stage is recomputed from the kernel's
own inputs to that stage -- the residual and skip GEMMs from the forward's zsave, dx / dhaux / the weight gradients
from the dpre the backward leaves in its workspace (z (B,T,R) then dpre (B,T,2R)) -- so a failure names one stage and,
through ``assert_within``, one 64-row time tile and 32-column group.

Semantics checked in every case: outputs and the workspace start as NaN inside sentinel margins that must survive;
gradient buffers start nonzero and got - init is what the bound covers (= where += belongs); without zsave the forward's
xout and skip are bit-identical to the run with zsave; with dout = NULL (last layer) dw2[:R] and db2[:R] stay
bit-identical; the fp32 post network leaves ``skip`` bitwise unchanged (the tensor-core forward rectifies it in place,
this one applies ReLU on load).

The cases reach the tiling edges of gemm_simt (64-row time tiles, 128-row M tiles, K streamed in chunks of 16, 64-channel
gate passes):

| case | R | S | Ap | ks | d | B, T | reaches |
|---|---|---|---|---|---|---|---|
| tiny | 4 | 1 | 32 | 1 | 1 | 1, 1 | one row, one 64-channel pass with 60 empty channels, M2 = 5 |
| dT-1 | 24 | 96 | 80 | 2 | T - 1 | 3, 63 | K1 = 128 (8 chunks), d = T - 1, one partial time tile |
| last | 100 | 250 | 32 | 3 | 70 >= T | 1, 65 | two gate passes (the second of 36), M2 = 350 (3 M tiles), last layer |
| recipe | 512 | 256 | 80 | 2 | 16 | 1, 1000 | 8 gate passes, 149 KB of dynamic shared memory, 16 time tiles |
| ks4 | 100 | 512 | 256 | 4 | 3 | 3, 1000 | ks = 4, Ap = 256, K1 = 656 (41 chunks), S = 512 |
| wide | 512 | 96 | 32 | 4 | 1000 >= T | 1, 63 | R = 512, ks = 4 with every older tap in the causal zero fill, last layer |
| max | largest R | 1 | 32 | 1 | 1 | 1, 65 | the largest R wnb_resblock_fwd_supported(FP32) accepts (R + 1 rejected) |

The largest err/bound of every stage is printed and, when $WNB_PARITY_OUT is set, written there as tc_stages_*.json.
"""
import math

import pytest
import torch

from tests import tc_reference as ref
from tests.test_gpu_tc_stages import Guarded, Log, _report

pytestmark = pytest.mark.gpu

FP32 = dict(cv=ref.exact, gate_fn=ref.GATE_LIBM)


def _lib():
    from pytorchwavenetvocoder_b200 import _lib as L
    return L, L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tn_slots(B, T, tiles):
    """partial sums gemm_tn adds per weight-gradient element: one per (batch, time range) (mirrors pick_tchunk)"""
    nsplit = max(1, -(-_sms() * 2 // (tiles * B)))
    chunk = max(64, -(-(-(-T // nsplit)) // 16) * 16)
    return B * -(-T // chunk)


def _nsm(B, T, M, N):
    """partial sums per element of a weight gradient (M x N, several launches) and of its bias (rows of 512)"""
    return max(_tn_slots(B, T, -(-M // 128) * -(-N // 64)), -(-(B * T) // 512))


def _max_fp32_r(lib, L_):
    R_ = 64
    while lib.wnb_resblock_fwd_supported(R_ + 1, 1, 32, 1, L_.MATH_FP32):
        R_ += 1
    return R_


def _perblock_fp32(R_, S, Ap, ks, d, B, T, last, init, seed):
    L_, lib = _lib()
    assert lib.wnb_resblock_fwd_supported(R_, S, Ap, ks, L_.MATH_FP32) == 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    K1 = ks * R_ + Ap
    xin, haux = rn(B, T, R_), rn(B, T, Ap)
    w1, b1 = 2 * rn(2 * R_, K1) / math.sqrt(K1), 0.2 * rn(2 * R_)
    w2, b2 = rn(R_ + S, R_) / math.sqrt(R_), 0.1 * rn(R_ + S)
    G = Guarded()
    skip0 = rn(B, T, S)
    skip = G((B, T, S), skip0)
    xout = None if last else G((B, T, R_))
    zsave = G((B, T, R_))
    args = lambda xo, sk, zs: (L_.ptr(xin), L_.ptr(haux), L_.ptr(w1), L_.ptr(b1), L_.ptr(w2), L_.ptr(b2),   # noqa: E731
                               L_.ptr(xo), L_.ptr(sk), L_.ptr(zs), B, T, R_, S, Ap, ks, d, 1 if init else 0,
                               L_.MATH_FP32, L_.stream())
    L_.check(lib.wnb_resblock_fwd(*args(xout, skip, zsave)), "resblock_fwd")
    # the same forward without zsave: z stays on chip, xout and skip must not change by a bit
    skip_nz = G((B, T, S), skip0)
    xout_nz = None if last else G((B, T, R_))
    L_.check(lib.wnb_resblock_fwd(*args(xout_nz, skip_nz, None)), "resblock_fwd (no zsave)")
    # backward with the same operands
    dout = None if last else rn(B, T, R_)
    dskip = rn(B, T, S)
    w1t, w2t = w1.t().contiguous(), w2.t().contiguous()
    ginit = dict(dh=rn(B, T, Ap), dw1=rn(2 * R_, K1), db1=rn(2 * R_), dw2=rn(R_ + S, R_), db2=rn(R_ + S))
    gout = {k: G(tuple(v.shape), v) for k, v in ginit.items()}
    dx = G((B, T, R_))
    ws = G((lib.wnb_resblock_bwd_workspace(B, T, R_, S, Ap, ks) // 4,))
    L_.check(lib.wnb_resblock_bwd(L_.ptr(xin), L_.ptr(haux), L_.ptr(dout), L_.ptr(dskip), L_.ptr(w1), L_.ptr(b1),
                                  L_.ptr(w1t), L_.ptr(w2t), L_.ptr(dx), L_.ptr(gout["dh"]), L_.ptr(gout["dw1"]),
                                  L_.ptr(gout["db1"]), L_.ptr(gout["dw2"]), L_.ptr(gout["db2"]), L_.ptr(ws),
                                  B, T, R_, S, Ap, ks, d, L_.MATH_FP32, L_.stream()), "resblock_bwd")
    torch.cuda.synchronize()
    G.check()
    log = Log()
    # ---- forward ----
    z_ref, e_z = ref.gate_fwd(xin, haux, w1, b1, d, ks, **FP32)
    log("z", zsave, (z_ref, e_z))
    if not last:
        log("xout", xout, ref.res_out(xin, zsave, w2[:R_], b2[:R_], cv=ref.exact))
        assert torch.equal(xout_nz, xout), "xout differs without zsave"
    log("skip", skip, ref.skip_gemm(zsave, w2[R_:], b2[R_:], False, cv=ref.exact, skip_in=None if init else skip0))
    assert torch.equal(skip_nz, skip), "skip differs without zsave"
    # ---- backward: workspace = z (B,T,R) | dpre (B,T,2R) ----
    zb = ws[:B * T * R_].view(B, T, R_)
    dpre = ws[B * T * R_:].view(B, T, 2 * R_)
    log("z(bwd)", zb, (z_ref, e_z))
    dz, e_dz = ref.dz_perblock(dout, dskip, w2, cv=ref.exact)
    log("dpre", dpre, ref.gate_bwd(xin, haux, w1, b1, d, ks, dz, e_dz, **FP32))
    log("dx", dx, ref.dx_stage(dpre, w1, d, ks, dout, cv=ref.exact))
    log("dhaux", gout["dh"], ref.accumulate(ginit["dh"], [ref.dhaux_stage(dpre, w1, ks, cv=ref.exact)]))
    nsm = _nsm(B, T, 2 * R_, max(R_, Ap))
    (dw, bw), (db, bb) = ref.wgrad(dpre, ref.taps(xin, ks, d) + [haux], ginit["dw1"], ginit["db1"], cv=ref.exact, nsm=nsm)
    log("dW1", gout["dw1"], (dw, bw))
    log("db1", gout["db1"], (db, bb))
    r0 = R_ if last else 0
    a = dskip if last else torch.cat([dout, dskip], -1)
    nsm = _nsm(B, T, max(R_, S), R_)
    (dw, bw), (db, bb) = ref.wgrad(a, [zb], ginit["dw2"][r0:], ginit["db2"][r0:], cv=ref.exact, nsm=nsm)
    log("dW2", gout["dw2"][r0:], (dw, bw))
    log("db2", gout["db2"][r0:], (db, bb))
    if last:
        assert torch.equal(gout["dw2"][:R_], ginit["dw2"][:R_]) and torch.equal(gout["db2"][:R_], ginit["db2"][:R_])
    _report("fp32_perblock_R%d_S%d_Ap%d_ks%d_d%d_B%d_T%d%s%s" % (R_, S, Ap, ks, d, B, T, "_last" if last else "",
                                                                  "_init" if init else ""), log.res)
    return log.res


@pytest.mark.parametrize("R_,S,Ap,ks,d,B,T,last,init", [
    (4, 1, 32, 1, 1, 1, 1, False, True),
    (24, 96, 80, 2, 62, 3, 63, False, False),
    (100, 250, 32, 3, 70, 1, 65, True, True),
    (512, 256, 80, 2, 16, 1, 1000, False, False),
    (100, 512, 256, 4, 3, 3, 1000, False, True),
    (512, 96, 32, 4, 1000, 1, 63, True, False),
], ids=["tiny", "dT-1", "last", "recipe", "ks4", "wide"])
def test_fp32_block_fwd_bwd(R_, S, Ap, ks, d, B, T, last, init):
    _perblock_fp32(R_, S, Ap, ks, d, B, T, last, init, seed=R_ + S + Ap + ks + d + T)


def test_fp32_block_largest_r():
    """the largest R the SIMT forward's shared-memory gate tile allows; R + 1 is rejected before any launch"""
    L_, lib = _lib()
    R_ = _max_fp32_r(lib, L_)
    assert R_ >= 512
    assert lib.wnb_resblock_fwd_supported(R_ + 1, 1, 32, 1, L_.MATH_FP32) == 0
    x = torch.zeros(4, device="cuda")
    n0 = L_.launch_count()
    rc = lib.wnb_resblock_fwd(*([L_.ptr(x)] * 9), 1, 1, R_ + 1, 1, 32, 1, 1, 1, L_.MATH_FP32, L_.stream())
    assert rc == -1 and L_.launch_count() == n0, rc
    _perblock_fp32(R_, 1, 32, 1, 1, 1, 65, False, True, seed=R_)


# ------------------------------------------------------------------------------------------------------------------
# the post network in fp32, and the standalone causal conv
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,S,Q,rectified", [(1, 1, 1, 2, 0), (3, 65, 96, 256, 0), (1, 130, 250, 33, 1),
                                               (2, 63, 512, 256, 0)])
def test_fp32_post_network(B, T, S, Q, rectified):
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(B + T + S + Q)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    skip_in = rn(B, T, S)
    if rectified:
        skip_in = skip_in.clamp_min(0)
    wp1, bp1 = rn(S, S) / math.sqrt(S), 0.1 * rn(S)
    wp2, bp2 = rn(Q, S) / math.sqrt(S), 0.1 * rn(Q)
    G = Guarded()
    skip = G((B, T, S), skip_in)
    r1, logits = G((B, T, S)), G((B, T, Q))
    L_.check(lib.wnb_post_fwd(L_.ptr(skip), L_.ptr(wp1), L_.ptr(bp1), L_.ptr(wp2), L_.ptr(bp2), L_.ptr(r1),
                              L_.ptr(logits), B, T, S, Q, L_.MATH_FP32, rectified, L_.stream()), "post_fwd")
    dlogits = rn(B, T, Q) / (B * T)
    init = dict(dwp1=rn(S, S), dbp1=rn(S), dwp2=rn(Q, S), dbp2=rn(Q))
    out = {k: G(tuple(v.shape), v) for k, v in init.items()}
    dskip, ws = G((B, T, S)), G((B, T, S))
    wp1t, wp2t = wp1.t().contiguous(), wp2.t().contiguous()
    L_.check(lib.wnb_post_bwd(L_.ptr(skip), L_.ptr(r1), L_.ptr(dlogits), L_.ptr(wp1t), L_.ptr(wp2t), L_.ptr(dskip),
                              L_.ptr(out["dwp1"]), L_.ptr(out["dbp1"]), L_.ptr(out["dwp2"]), L_.ptr(out["dbp2"]),
                              L_.ptr(ws), B, T, S, Q, L_.MATH_FP32, L_.stream()), "post_bwd")
    torch.cuda.synchronize()
    G.check()
    assert torch.equal(skip, skip_in), "the fp32 post network must leave skip unchanged"
    log = Log()
    skip_r = skip_in.clamp_min(0)
    log("r1", r1, ref.skip_gemm(skip_r, wp1, bp1, True, cv=ref.exact))
    log("logits", logits, ref.skip_gemm(r1, wp2, bp2, False, cv=ref.exact))
    pb = ref.post_bwd(skip_r, r1, dlogits, ws, wp1, wp2, cv=ref.exact)
    log("dh1", ws, pb["dh1"])
    log("dskip", dskip, pb["dskip"])
    (dw, bw), (db, bb) = ref.wgrad(dlogits, [r1], init["dwp2"], init["dbp2"], cv=ref.exact, nsm=_nsm(B, T, Q, S))
    log("dwp2", out["dwp2"], (dw, bw))
    log("dbp2", out["dbp2"], (db, bb))
    (dw, bw), (db, bb) = ref.wgrad(ws, [skip_r], init["dwp1"], init["dbp1"], cv=ref.exact, nsm=_nsm(B, T, S, S))
    log("dwp1", out["dwp1"], (dw, bw))
    log("dbp1", out["dbp1"], (db, bb))
    _report("fp32_post_B%d_T%d_S%d_Q%d" % (B, T, S, Q), log.res)


@pytest.mark.parametrize("B,T,Cin,Cout,ks,d,bias", [(2, 65, 28, 64, 1, 1, True), (1, 63, 3, 100, 2, 62, True),
                                                    (3, 130, 64, 512, 3, 7, False), (1, 10, 5, 7, 4, 20, True)])
def test_fp32_causal_conv1d(B, T, Cin, Cout, ks, d, bias):
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(B + T + Cin + ks)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    x = rn(B, T, Cin)
    w = rn(Cout, ks * Cin) / math.sqrt(ks * Cin)
    b = 0.1 * rn(Cout) if bias else None
    G = Guarded()
    out = G((B, T, Cout))
    L_.check(lib.wnb_causal_conv1d_fwd(L_.ptr(x), L_.ptr(w), L_.ptr(b), L_.ptr(out), B, T, Cin, Cout, ks, d,
                                       L_.stream()), "causal_conv1d_fwd")
    torch.cuda.synchronize()
    G.check()
    log = Log()
    # the conv is gate_pre without an aux part: sum_j x(t - (ks-1-j) d) w[:, tap j]^T + bias
    want = ref.gate_pre(x, x.new_zeros(B, T, 0), w, b if bias else torch.zeros(Cout, device="cuda"), d, ks, ref.exact)
    log("conv", out, want)
    _report("fp32_conv_B%d_T%d_Cin%d_Cout%d_ks%d_d%d" % (B, T, Cin, Cout, ks, d), log.res)
