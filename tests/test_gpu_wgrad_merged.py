# -*- coding: utf-8 -*-
"""GPU tier: the stack's weight gradients (dW1, dW2res, dWskip and their biases), which wnb_stack_bwd runs as ONE
problem list in one launch over every SM, against float64 element by element.

The forward and backward run once per case; each weight gradient is then recomputed in float64 from the kernel's own
inputs (the workspace's dpre_l and dx_l, Z_all, dskip) and compared with tests/tc_reference.py's wgrad bound.  A second
backward from the same inputs must give bit-identical gradients (each problem's time chunks are fixed, each is summed
from zero by one CTA, and the reduce adds them in chunk order).

| case | L | S | B, T | reaches |
|---|---|---|---|---|
| one | 1 | 32 | 2, 20 | no dW2res problems, T < 32: one stage per batch row, fewer stages than SMs |
| deep | 64 | 256 | 1, 200 | 64 dW1 + 63 dW2res + 64 dWskip problems: more than one launch's problem table |
| wide | 5 | 512 | 3, 1040 | 4 dWskip M-blocks, time chunks spanning batch rows (33 stages per row) |
| bench | 30 | 256 | 2, 2100 | the bench depth: CTAs run chunks of several dW1 / dW2res segments after their dWskip chunk |
"""
import ctypes
import math

import pytest
import torch

from tests import tc_reference as ref
from tests.test_gpu_tc_stages import AP, KS, R, Guarded, Log, _lib, _report, stack_bwd_workspace_views

pytestmark = pytest.mark.gpu

CASES = {"one": (1, 32, 2, 20), "deep": (64, 256, 1, 200), "wide": (5, 512, 3, 1040), "bench": (30, 256, 2, 2100)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_merged_weight_gradients(case):
    L_, lib = _lib()
    L, S, B, T = CASES[case]
    dil = [2 ** (i % 10) for i in range(L)]
    assert lib.wnb_stack_supported(R, S, AP, KS, L, L_.MATH_TF32)
    K1 = KS * R + AP
    g = torch.Generator(device="cuda").manual_seed(4242 + L + S + T)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    w1 = rn(L, 2 * R, K1) / math.sqrt(K1)
    b1 = 0.2 * rn(L, 2 * R)
    w2res = rn(L, R, R) / math.sqrt(R)
    b2res = 0.1 * rn(L, R)
    wskip = rn(S, L * R) / math.sqrt(L * R)
    bskip = 0.1 * rn(S)
    haux = rn(B, T, AP)
    xs = torch.empty(L, B, T, R, device="cuda")
    xs[0] = rn(B, T, R)
    zall, skip = torch.empty(B, T, L * R, device="cuda"), torch.empty(B, T, S, device="cuda")
    dils = (ctypes.c_int * L)(*dil)
    L_.check(lib.wnb_stack_fwd(L_.ptr(xs), L, L_.ptr(haux), L_.ptr(w1), L_.ptr(b1), L_.ptr(w2res), L_.ptr(b2res),
                               L_.ptr(wskip), L_.ptr(bskip), L_.ptr(zall), L_.ptr(skip), dils, L, B, T, R, S, AP, KS,
                               0, L_.stream()), "stack_fwd")
    dskip = rn(B, T, S)
    w1t = w1.transpose(1, 2).contiguous()
    wgate = torch.zeros(L, 3 * R, K1 + R, device="cuda")
    wgate[:, :2 * R, :K1] = w1
    wgate[:, 2 * R:, K1:] = w2res.transpose(1, 2)
    wskt = wskip.t().contiguous()
    init = dict(dhaux=rn(B, T, AP), dw1=rn(L, 2 * R, K1), db1=rn(L, 2 * R), dw2res=rn(L, R, R), db2res=rn(L, R),
                dwskip=rn(S, L * R), dbskip=rn(S))
    names = ("dw1", "db1", "dw2res", "db2res", "dwskip", "dbskip")

    def backward():
        G = Guarded()
        out = {k: G(tuple(v.shape), v) for k, v in init.items()}
        dx0 = G((B, T, R))
        ws = G((lib.wnb_stack_bwd_workspace(L, B, T, R, S, AP, KS) // 4,))
        L_.check(lib.wnb_stack_bwd(L_.ptr(xs), L_.ptr(haux), L_.ptr(zall), L_.ptr(dskip), L_.ptr(w1), L_.ptr(b1),
                                   L_.ptr(w1t), L_.ptr(wgate), L_.ptr(wskt), L_.ptr(dx0), L_.ptr(out["dhaux"]),
                                   L_.ptr(out["dw1"]), L_.ptr(out["db1"]), L_.ptr(out["dw2res"]), L_.ptr(out["db2res"]),
                                   L_.ptr(out["dwskip"]), L_.ptr(out["dbskip"]), L_.ptr(ws), dils, L, B, T, R, S, AP,
                                   KS, L_.stream()), "stack_bwd")
        torch.cuda.synchronize()
        G.check()
        return out, ws

    out, ws = backward()
    W = stack_bwd_workspace_views(ws, L, B, T, R)
    log = Log()
    for l in range(L):
        (dw, bw), (db, bb) = ref.wgrad(W["dpre"][l], ref.taps(xs[l], KS, dil[l]) + [haux], init["dw1"][l],
                                       init["db1"][l])
        log("dW1[block %d]" % l, out["dw1"][l], (dw, bw))
        log("db1[block %d]" % l, out["db1"][l], (db, bb))
        if l + 1 < L:
            (dw, bw), (db, bb) = ref.wgrad(W["dx"][l + 1], [zall[:, :, l * R:(l + 1) * R]], init["dw2res"][l],
                                           init["db2res"][l])
            log("dW2res[block %d]" % l, out["dw2res"][l], (dw, bw))
            log("db2res[block %d]" % l, out["db2res"][l], (db, bb))
    assert torch.equal(out["dw2res"][L - 1], init["dw2res"][L - 1]) and torch.equal(out["db2res"][L - 1],
                                                                                      init["db2res"][L - 1])
    (dw, bw), (db, bb) = ref.wgrad(dskip, [zall], init["dwskip"], init["dbskip"])
    log("dWskip", out["dwskip"], (dw, bw))
    log("dbskip", out["dbskip"], (db, bb))
    _report("wgrad_merged_%s_L%d_S%d_B%d_T%d" % (case, L, S, B, T), log.res)

    again, _ = backward()
    for k in names:
        assert torch.equal(out[k], again[k]), "%s differs between two identical backward calls" % k
