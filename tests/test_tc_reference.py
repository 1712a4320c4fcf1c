# -*- coding: utf-8 -*-
"""CPU tier: the float64 stage reference of tests/tc_reference.py is the model, its bounds are sound, and they are tight
enough to catch the faults tiled kernels make.

* Composing the stage functions (without tf32 conversion) over a small model reproduces oracle.wavenet_oracle's forward
  and backward to 1e-10: the reference implements WaveNet, not a look-alike.
* Soundness: a float32 emulation of the kernels' arithmetic (tf32 operands, fp32 accumulation in shuffled chunk
  orders, tanh perturbed by up to 2^-11 relative) stays inside the bounds over a few hundred seeded draws.
* Sensitivity: faults planted into otherwise exact results at the stage-test shapes are reported by assert_within,
  which names the tile.
* The same two checks for the fp32 (SIMT) model (cv=exact, gate_fn=GATE_LIBM): a float32 emulation of the SIMT kernels
  (one sequential fmaf per term, bias and epilogue roundings in kernel order, weight gradients summed per (batch, time
  range) slot and the slots in order, expf / tanhf off by up to 2 ulp) stays inside the bounds, and the faults a tiled
  FFMA kernel makes (a dropped 16-term K chunk, time tile, gate pass, tap or time range) are reported.
"""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests import tc_reference as ref

F64 = torch.float64


# ------------------------------------------------------------------------------------------------------------------
# the reference composes to the oracle
# ------------------------------------------------------------------------------------------------------------------
def _pack(cfg, p):
    R, S, ks, A = cfg.n_resch, cfg.n_skipch, cfg.kernel_size, cfg.n_aux
    Ap = -(-A // 32) * 32
    L = len(cfg.dilations)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float64))   # noqa: E731
    w1 = torch.zeros(L, 2 * R, ks * R + Ap, dtype=F64)
    b1 = torch.zeros(L, 2 * R, dtype=F64)
    for l in range(L):
        for br, name in enumerate(("sigmoid", "tanh")):
            rows = slice(br * R, (br + 1) * R)
            W = t(p["dil_%s.%d.conv.weight" % (name, l)])
            for j in range(ks):
                w1[l, rows, j * R:(j + 1) * R] = W[:, :, j]
            w1[l, rows, ks * R:ks * R + A] = t(p["aux_1x1_%s.%d.weight" % (name, l)])[:, :, 0]
            b1[l, rows] = t(p["dil_%s.%d.conv.bias" % (name, l)]) + t(p["aux_1x1_%s.%d.bias" % (name, l)])
    w2res = torch.stack([t(p["res_1x1.%d.weight" % l])[:, :, 0] for l in range(L)])
    b2res = torch.stack([t(p["res_1x1.%d.bias" % l]) for l in range(L)])
    wskip = torch.cat([t(p["skip_1x1.%d.weight" % l])[:, :, 0] for l in range(L)], 1)
    bskip = sum(t(p["skip_1x1.%d.bias" % l]) for l in range(L))
    post = [t(p["conv_post_1.weight"])[:, :, 0], t(p["conv_post_1.bias"]), t(p["conv_post_2.weight"])[:, :, 0],
            t(p["conv_post_2.bias"])]
    return Ap, w1, b1, w2res, b2res, wskip, bskip, post


@pytest.mark.parametrize("B,T", [(1, 1), (2, 37), (3, 70)])
def test_stages_compose_to_the_oracle(B, T):
    cfg = O.Config(64, 28, 64, 96, 4, 1, 2, 0)
    p = {k: v.astype(np.float64) for k, v in O.make_params(cfg, 5).items()}
    rng = np.random.RandomState(B * 100 + T)
    x = rng.randint(0, 64, size=(B, T)).astype(np.int64)
    h = rng.standard_normal((B, 28, T))
    y, cache = O.forward(cfg, p, x, h, return_cache=True)
    Ap, w1, b1, w2res, b2res, wskip, bskip, (wp1, bp1, wp2, bp2) = _pack(cfg, p)
    L, R, ks, cv = len(cfg.dilations), cfg.n_resch, cfg.kernel_size, ref.exact
    haux = torch.zeros(B, T, Ap, dtype=F64)
    haux[:, :, :28] = torch.from_numpy(h).transpose(1, 2)
    xs = [torch.from_numpy(cache["xs"][0]).transpose(1, 2).contiguous()]
    zs = []
    for l, d in enumerate(cfg.dilations):
        zs.append(ref.gate_fwd(xs[l], haux, w1[l], b1[l], d, ks, cv)[0])
        xs.append(ref.res_out(xs[l], zs[l], w2res[l], b2res[l], cv=cv)[0])
    zall = torch.cat(zs, -1)
    skip = ref.skip_gemm(zall, wskip, bskip, True, cv=cv)[0]
    (r1, _), logits_of = ref.post_fwd(skip, wp1, bp1, wp2, bp2, cv)
    logits = logits_of(r1)[0]
    assert np.abs(logits.numpy() - y).max() < 1e-10
    # backward from the oracle's dlogits
    loss, dl = O.cross_entropy(y, rng.randint(0, 64, size=(B, T)), 0)
    dl = torch.from_numpy(dl)
    pb = ref.post_bwd(skip, r1, dl, None, wp1, wp2, cv)
    g = O.backward(cfg, p, cache, dl.numpy())
    want = lambda k: torch.from_numpy(np.asarray(g[k], dtype=np.float64))   # noqa: E731
    got = {"conv_post_2.weight": pb["dwp2"][0], "conv_post_2.bias": pb["dbp2"][0],
           "conv_post_1.weight": pb["dwp1"][0], "conv_post_1.bias": pb["dbp1"][0]}
    dskip = pb["dskip"][0]
    dzall = ref.dz_all(dskip, wskip, cv)[0]
    dws, dbs = ref.wgrad(dskip, [zall], cv=cv)
    dout = None
    for l in reversed(range(L)):
        d = cfg.dilations[l]
        dz = ref.dz_block(dzall[:, :, l * R:(l + 1) * R], dout, w2res[l], cv)[0]
        dpre = ref.gate_bwd(xs[l], haux, w1[l], b1[l], d, ks, dz, 0 * dz, cv)[0]
        (dw1, _), (db1, _) = ref.wgrad(dpre, ref.taps(xs[l], ks, d) + [haux], cv=cv)
        if dout is not None:
            (dw2, _), (db2, _) = ref.wgrad(dout, [zs[l]], cv=cv)
            got["res_1x1.%d.weight" % l], got["res_1x1.%d.bias" % l] = dw2, db2
        for br, name in enumerate(("sigmoid", "tanh")):
            rows = slice(br * R, (br + 1) * R)
            got["dil_%s.%d.conv.weight" % (name, l)] = torch.stack([dw1[rows, j * R:(j + 1) * R] for j in range(ks)], -1)
            got["aux_1x1_%s.%d.weight" % (name, l)] = dw1[rows, ks * R:ks * R + 28]
            got["dil_%s.%d.conv.bias" % (name, l)] = db1[rows]
            got["aux_1x1_%s.%d.bias" % (name, l)] = db1[rows]
        got["skip_1x1.%d.weight" % l] = dws[0][:, l * R:(l + 1) * R]
        got["skip_1x1.%d.bias" % l] = dbs[0]
        dout = ref.dx_stage(dpre, w1[l], d, ks, dout, cv)[0]
    got["causal.conv.bias"] = dout.sum((0, 1))
    assert np.abs(g["res_1x1.%d.weight" % (L - 1)]).max() == 0      # the last block's residual output is unused
    for k, v in got.items():
        w = want(k).reshape(v.shape)
        assert (v - w).abs().max().item() <= 1e-10 * (1 + w.abs().max().item()), k


# ------------------------------------------------------------------------------------------------------------------
# float32 emulation of the kernels' arithmetic
# ------------------------------------------------------------------------------------------------------------------
class Emu:
    """tf32 operands, exact products, fp32 accumulation over a shuffled K in chunks of 8 (the per-k8 MMA) summed in
    fp32 in shuffled order; tanh.approx as tanh * (1 + delta), |delta| <= 2^-11"""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def mm(self, a, w):
        """a (..., K) @ w (N, K)^T"""
        A = ref.to_tf32(a.float()).reshape(-1, a.shape[-1])
        Wt = ref.to_tf32(w.float())
        P = (A[:, None, :] * Wt[None, :, :]).float()          # exact
        K = P.shape[-1]
        P = P[..., torch.randperm(K, generator=self.g)]
        chunks = []
        for c0 in range(0, K, 8):
            acc = torch.zeros(P.shape[:2], dtype=torch.float32)
            for k in range(c0, min(K, c0 + 8)):
                acc = acc + P[..., k]
            chunks.append(acc)
        acc = torch.zeros(P.shape[:2], dtype=torch.float32)
        for i in torch.randperm(len(chunks), generator=self.g).tolist():
            acc = acc + chunks[i]
        return acc.reshape(*a.shape[:-1], w.shape[0])

    def tanh(self, x):
        dl = (torch.rand(x.shape, generator=self.g) * 2 - 1) * 2.0 ** -11
        return (torch.tanh(x.double()) * (1 + dl)).float()

    def pre(self, xin, haux, w1, b1, d, ks):
        a = torch.cat(ref.taps(xin, ks, d) + [haux], -1)
        return self.mm(a, w1) + b1

    def gates(self, pre):
        R = pre.shape[-1] // 2
        s = 0.5 * self.tanh(0.5 * pre[..., :R]) + 0.5
        th = self.tanh(pre[..., R:])
        return s, th


def _rand(g, *sh, scale=1.0):
    return torch.randn(*sh, generator=g, dtype=torch.float32) * scale


@pytest.mark.parametrize("seed", range(40))
def test_bounds_hold_under_emulated_kernel_arithmetic(seed):
    """8 stages per draw, 40 draws: 320 stage checks; the largest err/bound is printed."""
    g = torch.Generator().manual_seed(seed)
    em = Emu(seed)
    R, Ap, ks = 64, 32, [1, 2, 3][seed % 3]
    B, T, d, S = 2, [1, 13, 40][seed % 3], 1 + seed % 7, 96
    K1 = ks * R + Ap
    xin, haux = _rand(g, B, T, R), _rand(g, B, T, Ap)
    w1, b1 = _rand(g, 2 * R, K1, scale=K1 ** -0.5), _rand(g, 2 * R, scale=0.3)
    w2res, b2res = _rand(g, R, R, scale=R ** -0.5), _rand(g, R, scale=0.1)
    wskip, bskip = _rand(g, S, R, scale=0.2), _rand(g, S, scale=0.1)
    worst = 0.0
    # gate forward
    pre = em.pre(xin, haux, w1, b1, d, ks)
    s, th = em.gates(pre)
    z = s * th
    worst = max(worst, ref.assert_within(z, *ref.gate_fwd(xin, haux, w1, b1, d, ks), "z"))
    # residual output and skip from the emulated z
    xout = em.mm(z, w2res) + b2res + xin
    worst = max(worst, ref.assert_within(xout, *ref.res_out(xin, z, w2res, b2res), "xout"))
    sk = (em.mm(z, wskip) + bskip).clamp_min(0)
    worst = max(worst, ref.assert_within(sk, *ref.skip_gemm(z, wskip, bskip, True), "skip"))
    # dZ and the gate backward (dz = dZ + dout W2res)
    dskip, dout = _rand(g, B, T, S), _rand(g, B, T, R)
    dzl = em.mm(dskip, wskip.t().contiguous())
    worst = max(worst, ref.assert_within(dzl, *ref.dz_all(dskip, wskip), "dZ"))
    dz = dzl + em.mm(dout, w2res.t().contiguous())
    dz_ref, e_dz = ref.dz_block(dzl, dout, w2res)
    worst = max(worst, ref.assert_within(dz, dz_ref, e_dz, "dz"))
    s, th = em.gates(em.pre(xin, haux, w1, b1, d, ks))
    dpre = torch.cat([dz * th * s * (1 - s), dz * s * (1 - th * th)], -1)
    worst = max(worst, ref.assert_within(dpre, *ref.gate_bwd(xin, haux, w1, b1, d, ks, dz_ref, e_dz), "dpre"))
    # dx and the weight gradient from the emulated dpre
    dx = sum(em.mm(ref.tshift(dpre, (ks - 1 - j) * d), w1[:, j * R:(j + 1) * R].t().contiguous())
             for j in range(ks)) + dout
    worst = max(worst, ref.assert_within(dx, *ref.dx_stage(dpre, w1, d, ks, dout), "dx"))
    bm = torch.cat(ref.taps(xin, ks, d) + [haux], -1)
    init = _rand(g, 2 * R, K1)
    dw1 = em.mm(dpre.reshape(-1, 2 * R).t().contiguous(), bm.reshape(-1, K1).t().contiguous()) + init
    (dw, bw), _ = ref.wgrad(dpre, ref.taps(xin, ks, d) + [haux], init)
    worst = max(worst, ref.assert_within(dw1, dw, bw, "dW1"))
    print("seed %d: largest err/bound %.3f" % (seed, worst))


# ------------------------------------------------------------------------------------------------------------------
# planted faults are reported
# ------------------------------------------------------------------------------------------------------------------
_SHAPES = {"b": (3, 96, 2, 95, [1, 64, 200]), "c": (5, 512, 3, 1040, [1, 2, 4, 8, 16])}


def _model(case):
    L, S, B, T, dil = _SHAPES[case]
    g = torch.Generator().manual_seed(ord(case))
    R, Ap, K1 = 64, 32, 160
    m = dict(L=L, S=S, B=B, T=T, dil=dil, R=R, Ap=Ap, K1=K1)
    m["xs"] = _rand(g, L + 1, B, T, R)
    m["haux"] = _rand(g, B, T, Ap)
    m["w1"], m["b1"] = _rand(g, L, 2 * R, K1, scale=K1 ** -0.5), _rand(g, L, 2 * R, scale=0.2)
    m["wskip"], m["bskip"] = _rand(g, S, L * R, scale=(L * R) ** -0.5), _rand(g, S, scale=0.1)
    m["zall"] = torch.cat([ref.gate_fwd(m["xs"][l], m["haux"], m["w1"][l], m["b1"][l], dil[l], 2)[0].float()
                           for l in range(L)], -1)
    m["dskip"] = _rand(g, B, T, S)
    m["dpre"] = _rand(g, L, B, T, 2 * R, scale=0.1)
    m["init"] = _rand(g, L, 2 * R, K1)
    return m


def _raises(got, want, what, expect=None):
    with pytest.raises(AssertionError) as ei:
        ref.assert_within(got, want[0], want[1], what)
    msg = str(ei.value)
    assert "tile" in msg or "group" in msg, msg
    if expect:
        assert expect in msg, msg
    return msg


@pytest.mark.parametrize("case", ["b", "c"])
def test_planted_faults_are_reported(case):
    m = _model(case)
    L, B, T, R, Ap, dil = m["L"], m["B"], m["T"], m["R"], m["Ap"], m["dil"]
    l = 0
    x, haux, w1, b1 = m["xs"][l], m["haux"], m["w1"][l], m["b1"][l]
    zref = ref.gate_fwd(x, haux, w1, b1, dil[l], 2)
    # the unfaulted results pass
    ref.assert_within(zref[0], *zref, "z")
    # 1. the dilated tap shifted by one step
    _raises(ref.gate_fwd(x, haux, w1, b1, dil[l] + 1, 2)[0], zref, "z, tap shifted")
    # 2. the last partial time tile dropped
    bad = zref[0].clone()
    t0 = (T - 1) // 64 * 64
    bad[:, t0:] = 0
    _raises(bad, zref, "z, last tile dropped", "time tile %d" % (t0 // 64))
    # 3. one 32-row stage of a weight-gradient reduction dropped, or counted twice
    taps = ref.taps(x, 2, dil[l]) + [haux]
    want, _ = ref.wgrad(m["dpre"][l], taps, m["init"][l])
    for factor in (0.0, 2.0):
        a = m["dpre"][l].clone()
        a[B - 1, 32:64] *= factor
        _raises(ref.wgrad(a, taps, m["init"][l])[0][0], want, "dW1, stage x%g" % factor)
    # 4. two 32-column groups swapped
    sk = ref.skip_gemm(m["zall"], m["wskip"], m["bskip"], False)
    bad = sk[0].clone()
    bad[..., 0:32], bad[..., 32:64] = sk[0][..., 32:64], sk[0][..., 0:32]
    _raises(bad, sk, "skip, groups swapped", "column group")
    # 5. segment l reading segment l+1's batch
    wrong = ref.taps(m["xs"][l + 1], 2, dil[l]) + [haux]
    _raises(ref.wgrad(m["dpre"][l], wrong, m["init"][l])[0][0], want, "dW1, wrong segment")
    # 6. overwrite instead of accumulate
    _raises(ref.wgrad(m["dpre"][l], taps)[0][0], want, "dW1, overwritten")
    # 7. the dhaux columns of the shifted tap not zeroed: its segment adds dpre(t + d) W1[:, R:R+Ap] to dhaux
    dh = ref.dhaux_stage(m["dpre"][l], w1, 2)
    bad = dh[0] + ref.tshift(m["dpre"][l], dil[l]).double() @ w1[:, R:R + Ap].double()
    _raises(bad, dh, "dhaux, shifted tap not zeroed")
    # the skip GEMM and dZ_all see a wrong K block (segment l's slice of Z_all replaced by block l+1's)
    bad_z = m["zall"].clone()
    bad_z[..., 0:R] = m["zall"][..., R:2 * R]
    _raises(ref.skip_gemm(bad_z, m["wskip"], m["bskip"], False)[0], sk, "skip, wrong slice")


# ------------------------------------------------------------------------------------------------------------------
# the fp32 (SIMT) model: float32 emulation of the FFMA kernels
# ------------------------------------------------------------------------------------------------------------------
F32 = torch.float32


class EmuF32:
    """The SIMT kernels' arithmetic: every term added with one fmaf in K order (gemm_simt.cuh streams K in chunks of 16
    into one register accumulator), weight gradients per (batch, time range) slot with the slots added in order, expf /
    tanhf perturbed by up to 2 ulp (emulated fmaf: the float64 sum of an exact product is rounded twice, which only adds
    to the error the bounds must cover)."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    @staticmethod
    def fma_seq(a, b, acc=None):
        """acc + sum_k a[..., k] b[k, :] with one fmaf per k, k in order; a (M, K), b (K, N) float32"""
        a, b = a.double(), b.double()
        acc = torch.zeros(a.shape[0], b.shape[1], dtype=F32) if acc is None else acc
        for k in range(a.shape[1]):
            acc = (a[:, k:k + 1] * b[k:k + 1, :] + acc.double()).float()
        return acc

    def mm(self, a, w):
        """a (..., K) @ w (N, K)^T"""
        return self.fma_seq(a.reshape(-1, a.shape[-1]), w.t()).reshape(*a.shape[:-1], w.shape[0])

    def fn(self, exact64):
        """a libm result within 2 ulp of the exact value: round(exact + delta ulp), |delta| <= 1.5, half the draws at
        the extremes"""
        _, ex = torch.frexp(exact64)
        ulp = torch.ldexp(torch.ones_like(exact64), ex - 24)
        dl = (torch.rand(exact64.shape, generator=self.g, dtype=F64) * 2 - 1) * 1.5
        edge = torch.rand(exact64.shape, generator=self.g) < 0.5
        dl = torch.where(edge, dl.sign() * 1.5, dl)
        return (exact64 + dl * ulp).float()

    def gates(self, pre):
        R = pre.shape[-1] // 2
        e = self.fn(torch.exp(-pre[..., :R].double()))
        s = (1 / (1 + e.double()).float().double()).float()
        th = self.fn(torch.tanh(pre[..., R:].double()))
        return s, th

    def pre(self, xin, haux, w1, b1, d, ks):
        a = torch.cat(ref.taps(xin, ks, d) + [haux], -1)
        return self.mm(a, w1) + b1

    def wgrad(self, a, b, init, tchunk):
        """init + sum over slots (b, time range of tchunk) of a^T b, slots in order; a (B,T,M), b (B,T,N)"""
        B, T = a.shape[:2]
        total = None
        for bi in range(B):
            for t0 in range(0, T, tchunk):
                part = self.fma_seq(a[bi, t0:t0 + tchunk].t(), b[bi, t0:t0 + tchunk])
                total = part if total is None else total + part
        return init + total

    @staticmethod
    def colsum(a, init, rows_per_block=512):
        a = a.reshape(-1, a.shape[-1])
        total = None
        for r0 in range(0, a.shape[0], rows_per_block):
            s = torch.zeros(a.shape[1], dtype=F32)
            for r in range(r0, min(r0 + rows_per_block, a.shape[0])):
                s = s + a[r]
            total = s if total is None else total + s
        return init + total


_FP32_KW = dict(cv=ref.exact, gate_fn=ref.GATE_LIBM)


@pytest.mark.parametrize("seed", range(24))
def test_fp32_bounds_hold_under_emulated_simt_arithmetic(seed):
    """every fp32 stage per draw, 24 draws, from the emulated kernel's own inputs; the largest err/bound is printed"""
    g = torch.Generator().manual_seed(500 + seed)
    em = EmuF32(seed)
    R, Ap, ks = [24, 40, 20][seed % 3], [32, 16, 8][seed % 3], 1 + seed % 4
    B, T, d, S = 1 + seed % 2, [1, 9, 23][seed % 3], 1 + seed % 5, 36
    K1 = ks * R + Ap
    xin, haux = _rand(g, B, T, R), _rand(g, B, T, Ap)
    w1, b1 = _rand(g, 2 * R, K1, scale=2 * K1 ** -0.5), _rand(g, 2 * R, scale=0.3)
    w2, b2 = _rand(g, R + S, R, scale=R ** -0.5), _rand(g, R + S, scale=0.1)
    worst = 0.0
    # forward: z, the residual output and the skip accumulation from the emulated z
    s, th = em.gates(em.pre(xin, haux, w1, b1, d, ks))
    z = s * th
    worst = max(worst, ref.assert_within(z, *ref.gate_fwd(xin, haux, w1, b1, d, ks, **_FP32_KW), "z"))
    xout = (em.mm(z, w2[:R]) + b2[:R]) + xin
    worst = max(worst, ref.assert_within(xout, *ref.res_out(xin, z, w2[:R], b2[:R], cv=ref.exact), "xout"))
    skip0 = _rand(g, B, T, S)
    sk = skip0 + (em.mm(z, w2[R:]) + b2[R:])
    worst = max(worst, ref.assert_within(sk, *ref.skip_gemm(z, w2[R:], b2[R:], False, cv=ref.exact, skip_in=skip0),
                                         "skip"))
    # backward: dz = [dout | dskip] W2 in one K loop, the gate from a recomputed pre, dpre in kernel order
    dout, dskip = _rand(g, B, T, R), _rand(g, B, T, S)
    dz = em.mm(torch.cat([dout, dskip], -1), w2.t().contiguous())
    dz_ref, e_dz = ref.dz_perblock(dout, dskip, w2, cv=ref.exact)
    worst = max(worst, ref.assert_within(dz, dz_ref, e_dz, "dz"))
    s, th = em.gates(em.pre(xin, haux, w1, b1, d, ks))
    dpre = torch.cat([dz * th * s * (1 - s), dz * s * (1 - th * th)], -1)
    worst = max(worst, ref.assert_within(dpre, *ref.gate_bwd(xin, haux, w1, b1, d, ks, dz_ref, e_dz, **_FP32_KW),
                                         "dpre"))
    # dx: one K loop over the ks shifted taps of dpre, then + dout
    dx = em.mm(torch.cat([ref.tshift(dpre, (ks - 1 - j) * d) for j in range(ks)], -1),
               torch.cat([w1[:, j * R:(j + 1) * R].t() for j in range(ks)], -1)) + dout
    worst = max(worst, ref.assert_within(dx, *ref.dx_stage(dpre, w1, d, ks, dout, cv=ref.exact), "dx"))
    # weight and bias gradients: time ranges of tchunk (the kernel's are >= 64; shorter here so several slots add up)
    tchunk = [1, 4, 16][seed % 3]
    nsm = B * -(-T // tchunk)
    bm = torch.cat(ref.taps(xin, ks, d) + [haux], -1)
    init_w, init_b = _rand(g, 2 * R, K1), _rand(g, 2 * R)
    dw1 = em.wgrad(dpre, bm, init_w, tchunk)
    db1 = em.colsum(dpre, init_b, rows_per_block=[1, 5, 512][seed % 3])
    (dw, bw), (db, bb) = ref.wgrad(dpre, ref.taps(xin, ks, d) + [haux], init_w, init_b, cv=ref.exact, nsm=nsm)
    worst = max(worst, ref.assert_within(dw1, dw, bw, "dW1"))
    worst = max(worst, ref.assert_within(db1, db, bb, "db1"))
    print("seed %d: largest err/bound %.3f" % (seed, worst))


def _fp32_model():
    """a block at SIMT tiling edges: R = 100 (two 64-channel gate passes, the second partial), K1 = 3*100 + 80 = 380
    (23 full 16-term K chunks and a partial one), T = 130 (three 64-row time tiles, the last of 2 rows)"""
    g = torch.Generator().manual_seed(77)
    R, S, Ap, ks, B, T, d = 100, 96, 80, 3, 2, 130, 5
    K1 = ks * R + Ap
    m = dict(R=R, S=S, Ap=Ap, ks=ks, B=B, T=T, d=d, K1=K1)
    m["xin"], m["haux"] = _rand(g, B, T, R), _rand(g, B, T, Ap)
    m["w1"], m["b1"] = _rand(g, 2 * R, K1, scale=2 * K1 ** -0.5), _rand(g, 2 * R, scale=0.2)
    m["w2"], m["b2"] = _rand(g, R + S, R, scale=R ** -0.5), _rand(g, R + S, scale=0.1)
    m["dout"], m["dskip"] = _rand(g, B, T, R), _rand(g, B, T, S)
    m["init"] = _rand(g, 2 * R, K1)
    return m


def test_fp32_planted_faults_are_reported():
    m = _fp32_model()
    R, Ap, ks, B, T, d, K1 = m["R"], m["Ap"], m["ks"], m["B"], m["T"], m["d"], m["K1"]
    x, haux, w1, b1, w2, b2 = m["xin"], m["haux"], m["w1"], m["b1"], m["w2"], m["b2"]
    zref = ref.gate_fwd(x, haux, w1, b1, d, ks, **_FP32_KW)
    ref.assert_within(zref[0].float(), *zref, "z")
    # 1. the last (partial) 16-term K chunk dropped from the pre-activations
    w = w1.clone()
    w[:, K1 // 16 * 16:] = 0
    _raises(ref.gate_fwd(x, haux, w, b1, d, ks, **_FP32_KW)[0], zref, "z, last K chunk dropped")
    # 2. a dropped K chunk in the middle (the 16 channels of tap 1 starting at 112)
    w = w1.clone()
    w[:, 112:128] = 0
    _raises(ref.gate_fwd(x, haux, w, b1, d, ks, **_FP32_KW)[0], zref, "z, middle K chunk dropped")
    # 3. the second 64-channel gate pass reads the first pass's weight rows
    w = w1.clone()
    w[64:R], w[R + 64:] = w1[0:R - 64], w1[R:2 * R - 64]
    _raises(ref.gate_fwd(x, haux, w, b1, d, ks, **_FP32_KW)[0], zref, "z, gate pass 2", "ch=")
    # 4. the last partial time tile not written (left at the previous content, here 0)
    bad = zref[0].clone()
    bad[:, 128:] = 0
    _raises(bad, zref, "z, last time tile dropped", "time tile 2")
    # 5. tap 0 (the oldest) dropped: in the gate and in dx
    w = w1.clone()
    w[:, :R] = 0
    _raises(ref.gate_fwd(x, haux, w, b1, d, ks, **_FP32_KW)[0], zref, "z, tap 0 dropped")
    dz, e_dz = ref.dz_perblock(m["dout"], m["dskip"], w2, cv=ref.exact)
    dpre_ref = ref.gate_bwd(x, haux, w1, b1, d, ks, dz, e_dz, **_FP32_KW)
    _raises(ref.gate_bwd(x, haux, w, b1, d, ks, dz, e_dz, **_FP32_KW)[0], dpre_ref, "dpre, tap 0 dropped")
    dpre = dpre_ref[0].float()
    dxref = ref.dx_stage(dpre, w1, d, ks, m["dout"], cv=ref.exact)
    _raises(ref.dx_stage(dpre, w, d, ks, m["dout"], cv=ref.exact)[0], dxref, "dx, tap 0 dropped")
    # 6. dz without the dout rows (the last-layer K offset applied to an inner block)
    _raises(ref.dz_perblock(None, m["dskip"], w2, cv=ref.exact)[0], (dz, e_dz), "dz, dout rows skipped")
    # 7. the skip rows of W2 offset by one row
    skref = ref.skip_gemm(zref[0].float(), w2[R:], b2[R:], False, cv=ref.exact)
    _raises(ref.skip_gemm(zref[0].float(), w2[R - 1:-1], b2[R:], False, cv=ref.exact)[0], skref, "skip, row offset")
    # 8. the weight gradient without its last time range (T = 130: one range of 64 rows of batch 1, 2 rows short)
    taps = ref.taps(x, ks, d) + [haux]
    want, wb = ref.wgrad(dpre, taps, m["init"], cv=ref.exact, nsm=6)
    a = dpre.clone()
    a[B - 1, 128:] = 0
    _raises(ref.wgrad(a, taps, m["init"], cv=ref.exact)[0][0], want, "dW1, last time range dropped")
    with pytest.raises(AssertionError, match="db1, last row block dropped"):
        ref.assert_within(ref.wgrad(a, taps, m["init"], cv=ref.exact)[1][0], *wb, "db1, last row block dropped")
    # 9. one slot added twice
    a = dpre.clone()
    a[0, 64:128] *= 2
    _raises(ref.wgrad(a, taps, m["init"], cv=ref.exact)[0][0], want, "dW1, slot counted twice")
