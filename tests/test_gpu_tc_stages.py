# -*- coding: utf-8 -*-
"""GPU tier: every stage of the tf32 tensor-core training path against float64, element by element.

Teacher forcing.  ``wnb_stack_fwd`` (nxs = L, every block input kept) and ``wnb_stack_bwd`` run once per case; then each
stage is recomputed in float64 from the kernel's OWN inputs to that stage -- the forward from xs[l] and Z_all, the
backward from the workspace's dZ_all, dpre_l and dx_l (``stack_bwd_workspace_views``) -- and compared with the bound of
tests/tc_reference.py.  Every check is then a single-stage bound whatever the depth, and a failure names one block, one
launch and (through ``assert_within``) one 64-row time tile / 32-column group.

The cases reach the edges of the kernels' tiling (column 'reaches'):

| case | L | S | B, T | dilations | reaches |
|---|---|---|---|---|---|
| a | 1 | 32 | 1, 1 | 1 | a one-row tile, d >= T, no dW2res launch, ldz = 64 |
| b | 3 | 96 | 2, 95 | 1, 64, 200 | partial 64- and 32-row tiles, d > T, dWskip m_valid = 96 |
| c | 5 | 512 | 3, 1040 | 1..16 | dZ_all in five 64-column blocks, skip GEMM in 2 blocks, 4 dWskip M-blocks |
| d | 22 | 256 | 1, derived | mixed | weight-gradient CTAs with an empty time range in dW1, dW2res and dWskip |
| e | 30 | 512 | 2, 8300 | bench | several tiles per CTA in every kernel, reversed tile order on odd blocks |
| f | 64 | 128 | 1, 200 | mixed | 64 segments (the limit), dZ_all in 16 blocks, dWskip n_split = 32 |

Semantics checked in every case: gradient buffers start at nonzero values and got - init is compared (= where += belongs
fails); the last block's dW2res / db2res stay bit-identical; the workspace and every output start as NaN, so a read of
memory nothing wrote propagates; every output is a slice of a larger buffer whose sentinel margins must survive.

The largest err/bound of every stage is printed and, when $WNB_PARITY_OUT is set, written there as tc_stages_*.json.
"""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

from tests import stack_shapes as SS
from tests import tc_reference as ref

pytestmark = pytest.mark.gpu

R, AP, KS = 64, 32, 2
SENTINEL = 7777.0
PAD = 256   # floats of sentinel either side of an output (1 KB: keeps the 16-byte alignment TMA needs)


def _lib():
    from pytorchwavenetvocoder_b200 import _lib as L
    return L, L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Guarded:
    """outputs allocated as slices of sentinel-filled buffers"""

    def __init__(self):
        self.bufs = []

    def __call__(self, shape, fill=float("nan")):
        n = int(np.prod(shape))
        buf = torch.full((n + 2 * PAD,), SENTINEL, device="cuda")
        v = buf[PAD:PAD + n].view(*shape)
        if isinstance(fill, torch.Tensor):
            v.copy_(fill)
        else:
            v.fill_(fill)
        self.bufs.append(buf)
        return v

    def check(self):
        for i, b in enumerate(self.bufs):
            assert torch.all(b[:PAD] == SENTINEL) and torch.all(b[-PAD:] == SENTINEL), "write outside output %d" % i


def stack_bwd_workspace_views(ws, L, B, T, R):
    """The wnb_stack_bwd workspace on return (see wnb_stack_bwd_workspace in csrc/stack.cu):
    dZ_all (B,T,L*R), one row of slack, dpre of every block (L,B,T,2R), dx of every block (L,B,T,R) with slot 0 unused."""
    bt, ldz = B * T, L * R
    o = 0
    dzall = ws[o:o + bt * ldz].view(B, T, ldz); o += bt * ldz
    slack = ws[o:o + ldz]; o += ldz
    dpre = ws[o:o + L * bt * 2 * R].view(L, B, T, 2 * R); o += L * bt * 2 * R
    dx = ws[o:o + L * bt * R].view(L, B, T, R); o += L * bt * R
    assert o == ws.numel()
    return dict(dzall=dzall, slack=slack, dpre=dpre, dx=dx)


def _report(name, res):
    line = ", ".join("%s %.3g" % (k, v) for k, v in sorted(res.items()))
    print("largest err/bound [%s]: %s" % (name, line))
    d = os.environ.get("WNB_PARITY_OUT")
    if d:
        try:
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, "tc_stages_%s.json" % name), "w") as f:
                json.dump(res, f, indent=1, sort_keys=True)
        except OSError:
            pass


class Log:
    def __init__(self):
        self.res = {}

    def __call__(self, stage, got, want):
        r = ref.assert_within(got, want[0], want[1], stage)
        key = stage.split("[")[0]
        self.res[key] = max(self.res.get(key, 0.0), r)


# ------------------------------------------------------------------------------------------------------------------
# the deferred-skip stack, teacher-forced
# ------------------------------------------------------------------------------------------------------------------
def _dwskip_sets(L, S):
    groups = L * R // 32
    nB = next(c for c in range(7, 0, -1) if groups % c == 0 and groups // c <= 128)
    return ((S + 127) // 128) * (groups // nB)


def _has_empty_range(sets, ntiles, sms):
    k = min(max(1, sms // sets), ntiles)
    per = -(-ntiles // k)
    return any(min(ntiles, i * per) == min(ntiles, (i + 1) * per) for i in range(k))


def _empty_range_T(L, S, B, sms):
    """smallest T at which a CTA of each of the three segmented weight-gradient launches gets no time tile
    (mirrors the split of wgrad_tc_blocks: ksplit = min(SMs / CTA sets, tiles), per = ceil(tiles / ksplit))"""
    for T in range(1, 4000):
        nt = B * -(-T // 32)
        if all(_has_empty_range(s, nt, sms) for s in (L, L - 1, _dwskip_sets(L, S))):
            return T
    raise AssertionError("no T gives every weight-gradient launch an empty CTA range on %d SMs" % sms)


def _case(name):
    """the case's row of tests/stack_shapes.py; case d's T is the smallest that gives a weight-gradient CTA of each
    launch an empty time range on this device"""
    row = SS.STACK_ROWS["case_" + name]
    L, S, B, T = row["L"], row["S"], row["B"], row["T"]
    return L, S, B, (T if T is not None else _empty_range_T(L, S, B, _sms())), row["dilations"]


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("case", ["a", "b", "c", "d", "e", "f"])
def test_stack_stages(case, relu):
    L, S, B, T, dil = _case(case)
    _stack_stages(L, S, B, T, dil, relu, True, 1000 + ord(case) + relu,
                  "stack_%s_relu%d_L%d_S%d_B%d_T%d" % (case, relu, L, S, B, T))


def _stack_stages(L, S, B, T, dil, relu, aux, seed, name, repeat_bwd=False, check=True):
    """``wnb_stack_fwd`` + ``wnb_stack_bwd`` on random operands, every stage checked against float64 (check=False: run
    only).  aux=False: dhaux is NULL (a model without an up-sampling layer) and not checked.  repeat_bwd: a second
    backward from the same inputs must give bit-identical gradients and workspace.  Returns every output."""
    L_, lib = _lib()
    assert lib.wnb_stack_supported(R, S, AP, KS, L, L_.MATH_TF32)
    K1 = KS * R + AP
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    w1 = rn(L, 2 * R, K1) / math.sqrt(K1)
    b1 = 0.2 * rn(L, 2 * R)
    w2res = rn(L, R, R) / math.sqrt(R)
    b2res = 0.1 * rn(L, R)
    wskip = rn(S, L * R) / math.sqrt(L * R)
    bskip = 0.1 * rn(S)
    haux = rn(B, T, AP)
    G = Guarded()
    xs = G((L, B, T, R))
    xs[0] = rn(B, T, R)
    zall, skip = G((B, T, L * R)), G((B, T, S))
    dils = (ctypes.c_int * L)(*dil)
    L_.check(lib.wnb_stack_fwd(L_.ptr(xs), L, L_.ptr(haux), L_.ptr(w1), L_.ptr(b1), L_.ptr(w2res), L_.ptr(b2res),
                               L_.ptr(wskip), L_.ptr(bskip), L_.ptr(zall), L_.ptr(skip), dils, L, B, T, R, S, AP, KS,
                               relu, L_.stream()), "stack_fwd")
    # backward: nonzero initial gradients, NaN workspace and outputs
    dskip = rn(B, T, S)
    w1t = w1.transpose(1, 2).contiguous()
    wgate = torch.zeros(L, 3 * R, K1 + R, device="cuda")
    wgate[:, :2 * R, :K1] = w1
    wgate[:, 2 * R:, K1:] = w2res.transpose(1, 2)
    wskt = wskip.t().contiguous()
    init = dict(dhaux=rn(B, T, AP), dw1=rn(L, 2 * R, K1), db1=rn(L, 2 * R), dw2res=rn(L, R, R), db2res=rn(L, R),
                dwskip=rn(S, L * R), dbskip=rn(S))
    if not aux:
        del init["dhaux"]

    def backward():
        out = {k: G(tuple(v.shape), v) for k, v in init.items()}
        dx0 = G((B, T, R))
        ws = G((lib.wnb_stack_bwd_workspace(L, B, T, R, S, AP, KS) // 4,))
        L_.check(lib.wnb_stack_bwd(L_.ptr(xs), L_.ptr(haux), L_.ptr(zall), L_.ptr(dskip), L_.ptr(w1), L_.ptr(b1),
                                   L_.ptr(w1t), L_.ptr(wgate), L_.ptr(wskt), L_.ptr(dx0), L_.ptr(out.get("dhaux")),
                                   L_.ptr(out["dw1"]), L_.ptr(out["db1"]), L_.ptr(out["dw2res"]), L_.ptr(out["db2res"]),
                                   L_.ptr(out["dwskip"]), L_.ptr(out["dbskip"]), L_.ptr(ws), dils, L, B, T, R, S, AP, KS,
                                   L_.stream()), "stack_bwd")
        return out, dx0, ws
    out, dx0, ws = backward()
    if repeat_bwd:     # a second backward from the same inputs: bit-identical (fixed summation order)
        out2, dx02, ws2 = backward()
        assert torch.equal(dx02, dx0), "dx0 differs between two backward runs"
        assert torch.equal(ws2.nan_to_num(SENTINEL), ws.nan_to_num(SENTINEL)), "workspace differs between two runs"
        for k in out:
            assert torch.equal(out2[k], out[k]), "%s differs between two backward runs" % k
    torch.cuda.synchronize()
    G.check()
    result = dict(xs=xs, zall=zall, skip=skip, dx0=dx0, ws=ws, **out)
    if not check:
        return result
    W = stack_bwd_workspace_views(ws, L, B, T, R)
    log = Log()

    # ---- forward: gate of block l from xs[l]; residual output from xs[l] and the block's own Z_all slice ----
    for l in range(L):
        zl = zall[:, :, l * R:(l + 1) * R]
        log("z[block %d]" % l, zl, ref.gate_fwd(xs[l], haux, w1[l], b1[l], dil[l], KS))
        if l + 1 < L:
            log("xout[block %d]" % l, xs[l + 1], ref.res_out(xs[l], zl, w2res[l], b2res[l]))
    log("skip", skip, ref.skip_gemm(zall, wskip, bskip, relu))

    # ---- backward ----
    log("dZ_all", W["dzall"], ref.dz_all(dskip, wskip))
    assert torch.isnan(W["dx"][0]).all(), "dx slot 0 of the workspace is documented as unused"
    dh_parts = []
    for l in reversed(range(L)):
        d = dil[l]
        dout = W["dx"][l + 1] if l + 1 < L else None
        dz, e_dz = ref.dz_block(W["dzall"][:, :, l * R:(l + 1) * R], dout, w2res[l])
        log("dpre[block %d]" % l, W["dpre"][l], ref.gate_bwd(xs[l], haux, w1[l], b1[l], d, KS, dz, e_dz))
        log("dx[block %d]" % l, dx0 if l == 0 else W["dx"][l], ref.dx_stage(W["dpre"][l], w1[l], d, KS, dout))
        dh_parts.append(ref.dhaux_stage(W["dpre"][l], w1[l], KS))
        (dw, bw), (db, bb) = ref.wgrad(W["dpre"][l], ref.taps(xs[l], KS, d) + [haux], init["dw1"][l], init["db1"][l])
        log("dW1[block %d]" % l, out["dw1"][l], (dw, bw))
        log("db1[block %d]" % l, out["db1"][l], (db, bb))
        if l + 1 < L:
            (dw, bw), (db, bb) = ref.wgrad(W["dx"][l + 1], [zall[:, :, l * R:(l + 1) * R]], init["dw2res"][l],
                                           init["db2res"][l])
            log("dW2res[block %d]" % l, out["dw2res"][l], (dw, bw))
            log("db2res[block %d]" % l, out["db2res"][l], (db, bb))
    if aux:
        log("dhaux", out["dhaux"], ref.accumulate(init["dhaux"], dh_parts))
    assert torch.equal(out["dw2res"][L - 1], init["dw2res"][L - 1]) and torch.equal(out["db2res"][L - 1],
                                                                                      init["db2res"][L - 1])
    (dw, bw), (db, bb) = ref.wgrad(dskip, [zall], init["dwskip"], init["dbskip"])
    log("dWskip", out["dwskip"], (dw, bw))
    log("dbskip", out["dbskip"], (db, bb))
    _report(name, log.res)
    return result


# ------------------------------------------------------------------------------------------------------------------
# one block in deferred-skip form + the skip GEMM over a 3-block Z_all (only the block's slice is written)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,T,last", [(1, 256, False), (8, 1000, False), (512, 2048, False), (4, 300, True)])
def test_block_z_and_skip_gemm(d, T, last):
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(d + T)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    B, S, L, slot = 2, 512, 3, 1
    K1 = KS * R + AP
    xin, haux = rn(B, T, R), rn(B, T, AP)
    w1, b1 = rn(2 * R, K1) / math.sqrt(K1), 0.1 * rn(2 * R)
    w2res, b2res = rn(R, R) / math.sqrt(R), 0.1 * rn(R)
    G = Guarded()
    zall = G((B, T, L * R), SENTINEL)
    xout = None if last else G((B, T, R))
    L_.check(lib.wnb_resblock_fwd_z(L_.ptr(xin), L_.ptr(haux), L_.ptr(w1), L_.ptr(b1), L_.ptr(w2res), L_.ptr(b2res),
                                    L_.ptr(xout), L_.ptr(zall), L * R, slot * R, B, T, R, AP, KS, d, L_.stream()),
             "resblock_fwd_z")
    torch.cuda.synchronize()
    assert torch.all(zall[:, :, :slot * R] == SENTINEL) and torch.all(zall[:, :, (slot + 1) * R:] == SENTINEL)
    zall[:, :, :slot * R] = 0
    zall[:, :, (slot + 1) * R:] = rn(B, T, (L - slot - 1) * R)
    wskip, bskip = rn(S, L * R) / math.sqrt(L * R), 0.1 * rn(S)
    skip = G((B, T, S))
    L_.check(lib.wnb_skip_gemm(L_.ptr(zall), L_.ptr(wskip), L_.ptr(bskip), L_.ptr(skip), B, T, L * R, S, 0,
                               L_.stream()), "skip_gemm")
    torch.cuda.synchronize()
    G.check()
    log = Log()
    zl = zall[:, :, slot * R:(slot + 1) * R]
    log("z", zl, ref.gate_fwd(xin, haux, w1, b1, d, KS))
    if not last:
        log("xout", xout, ref.res_out(xin, zl, w2res, b2res))
    log("skip", skip, ref.skip_gemm(zall, wskip, bskip, 0))
    _report("block_z_d%d_T%d%s" % (d, T, "_last" if last else ""), log.res)


# ------------------------------------------------------------------------------------------------------------------
# per-block tf32 entries: the fused kernel (R = 64) and the composed path
# ------------------------------------------------------------------------------------------------------------------
def _perblock(R_, S, Ap, ks, d, B, T, last, init, seed, repeat_bwd=False, dhaux=True):
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, device="cuda", generator=g)   # noqa: E731
    K1 = ks * R_ + Ap
    xin, haux = rn(B, T, R_), rn(B, T, Ap)
    w1, b1 = rn(2 * R_, K1) / math.sqrt(K1), 0.2 * rn(2 * R_)
    w2, b2 = rn(R_ + S, R_) / math.sqrt(R_), 0.1 * rn(R_ + S)
    kind = lib.wnb_resblock_fwd_supported(R_, S, Ap, ks, L_.MATH_TF32)
    G = Guarded()
    skip0 = rn(B, T, S)
    skip = G((B, T, S), skip0)
    xout = None if last else G((B, T, R_))
    zsave = G((B, T, R_)) if kind == 2 else None
    L_.check(lib.wnb_resblock_fwd(L_.ptr(xin), L_.ptr(haux), L_.ptr(w1), L_.ptr(b1), L_.ptr(w2), L_.ptr(b2),
                                  L_.ptr(xout), L_.ptr(skip), L_.ptr(zsave), B, T, R_, S, Ap, ks, d, 1 if init else 0,
                                  L_.MATH_TF32, L_.stream()), "resblock_fwd")
    # backward with the same operands
    dout = None if last else rn(B, T, R_)
    dskip = rn(B, T, S)
    w1t, w2t = w1.t().contiguous(), w2.t().contiguous()
    ginit = dict(dh=rn(B, T, Ap), dw1=rn(2 * R_, K1), db1=rn(2 * R_), dw2=rn(R_ + S, R_), db2=rn(R_ + S))
    if not dhaux:      # dhaux NULL: the backward computes no aux gradient
        del ginit["dh"]

    def backward():
        gout = {k: G(tuple(v.shape), v) for k, v in ginit.items()}
        dx = G((B, T, R_))
        ws = G((lib.wnb_resblock_bwd_workspace(B, T, R_, S, Ap, ks) // 4,))
        L_.check(lib.wnb_resblock_bwd(L_.ptr(xin), L_.ptr(haux), L_.ptr(dout), L_.ptr(dskip), L_.ptr(w1), L_.ptr(b1),
                                      L_.ptr(w1t), L_.ptr(w2t), L_.ptr(dx), L_.ptr(gout.get("dh")), L_.ptr(gout["dw1"]),
                                      L_.ptr(gout["db1"]), L_.ptr(gout["dw2"]), L_.ptr(gout["db2"]), L_.ptr(ws),
                                      B, T, R_, S, Ap, ks, d, L_.MATH_TF32, L_.stream()), "resblock_bwd")
        return gout, dx, ws
    gout, dx, ws = backward()
    if repeat_bwd:     # a second backward from the same inputs: bit-identical gradients (fixed summation order)
        g2, dx2, _ = backward()
        assert torch.equal(dx2, dx), "dx differs between two backward runs"
        for k in gout:
            assert torch.equal(g2[k], gout[k]), "%s differs between two backward runs" % k
    torch.cuda.synchronize()
    G.check()
    log = Log()
    z_ref, e_z = ref.gate_fwd(xin, haux, w1, b1, d, ks)
    if kind == 2:       # z is in memory: the residual and skip GEMMs are checked from the kernel's own z
        log("z", zsave, (z_ref, e_z))
        zin, ez = zsave, None
    else:               # the fused kernel keeps z on chip: its xout / skip bounds carry the propagated gate error e_z
        zin, ez = z_ref.float(), e_z
    if not last:
        log("xout", xout, ref.res_out(xin, zin, w2[:R_], b2[:R_], e_z=ez))
    log("skip", skip, ref.skip_gemm(zin, w2[R_:], b2[R_:], False, e_z=ez, skip_in=None if init else skip0))
    # backward: workspace = z (B,T,R) | dpre (B,T,2R); dz itself is overwritten, so dpre carries the dz GEMM bound
    zb = ws[:B * T * R_].view(B, T, R_)
    dpre = ws[B * T * R_:].view(B, T, 2 * R_)
    log("z(bwd)", zb, (z_ref, e_z))
    dz, e_dz = ref.dz_perblock(dout, dskip, w2)
    log("dpre", dpre, ref.gate_bwd(xin, haux, w1, b1, d, ks, dz, e_dz))
    log("dx", dx, ref.dx_stage(dpre, w1, d, ks, dout))
    if dhaux:
        log("dhaux", gout["dh"], ref.accumulate(ginit["dh"], [ref.dhaux_stage(dpre, w1, ks)]))
    (dw, bw), (db, bb) = ref.wgrad(dpre, ref.taps(xin, ks, d) + [haux], ginit["dw1"], ginit["db1"])
    log("dW1", gout["dw1"], (dw, bw))
    log("db1", gout["db1"], (db, bb))
    r0 = R_ if last else 0
    a = dskip if last else torch.cat([dout, dskip], -1)
    (dw, bw), (db, bb) = ref.wgrad(a, [zb], ginit["dw2"][r0:], ginit["db2"][r0:])
    log("dW2", gout["dw2"][r0:], (dw, bw))
    log("db2", gout["db2"][r0:], (db, bb))
    if last:
        assert torch.equal(gout["dw2"][:R_], ginit["dw2"][:R_]) and torch.equal(gout["db2"][:R_], ginit["db2"][:R_])
    _report("perblock_R%d_S%d_Ap%d_ks%d_d%d_B%d_T%d%s%s%s" % (R_, S, Ap, ks, d, B, T, "_last" if last else "",
                                                               "_init" if init else "", "" if dhaux else "_nodhaux"),
            log.res)
    return kind


@pytest.mark.parametrize("S,d,T,init,last", [
    (64, 1, 1, True, False), (192, 4, 63, False, False), (512, 70, 65, True, False), (512, 68, 63, False, True),
    (192, 512, 8300, False, False), (64, 3, 8300, True, True)])
def test_fused_block_fwd_bwd(S, d, T, init, last):
    """R = 64 with S a multiple of 64: the fused per-block kernel (z stays on chip), d up to T + 5."""
    assert _perblock(64, S, 32, 2, d, 2, T, last, init, seed=S + d + T) == 1


@pytest.mark.parametrize("S", [32, 96])
def test_r64_odd_skip_takes_composed_path(S):
    """R = 64 with S not a multiple of 64 is not covered by the fused kernel: the composed path runs it."""
    assert _perblock(64, S, 32, 2, 5, 2, 65, False, False, seed=S) == 2


@pytest.mark.parametrize("R_,S,Ap,ks,d,T,last,init", [
    (128, 256, 32, 2, 4, 300, False, True),
    (512, 256, 32, 2, 16, 520, False, False),
    (128, 64, 96, 3, 2, 260, False, False),
    (192, 64, 32, 3, 8, 200, True, False),
    (192, 256, 96, 1, 1, 97, False, True),
    (512, 64, 96, 1, 7, 33, True, True),
    (128, 256, 32, 3, 40, 65, False, False),
])
def test_composed_block_fwd_bwd(R_, S, Ap, ks, d, T, last, init):
    assert _perblock(R_, S, Ap, ks, d, 2, T, last, init, seed=R_ + S + T + ks) == 2
