# -*- coding: utf-8 -*-
"""CPU tier: the layer-by-layer checker of the bf16 decoder (tests/decode_bf16_layers.py) without a GPU.

A float32 emulation of the decoder at small shapes produces what the GPU test reads from the kernel: every layer's
queue bf16(x_l(t)), the codes and the fp32 logits.  It rounds to bf16 where the kernel does (aux, layer inputs, z,
relu(skip), relu(post-1)), accumulates every product as the tensor cores do (k16 steps in the kernel's K order, one
fp32 rounding per step, to nearest or toward zero at random), and evaluates expf and tanhf within 2 ulp (the correctly
rounded value moved by -1, 0 or +1 ulp at random).  The checker must accept a few hundred clean steps at kernel size 2
and 3, with and without up-sampling, and a recipe-width model (R = S = 256), and reject each planted fault of the
emulation at R = 16 and at R = 256.  The exact helpers (fmaf, bf16 neighbours) are checked against constructed cases."""
import fractions
import re

import numpy as np
import pytest
import torch

from tests import decode_bf16_layers as DL

F32 = torch.float32


def _model(ks, U, R=16, S=16, Q=32, A=5, dil=(1, 2, 4, 1), seed=0):
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(F32)
    L, Ap = len(dil), 32
    K = ks * R + A
    W1 = rn(L, 2 * R, ks * R + Ap, scale=1.5 / K ** 0.5)
    W1[:, :, ks * R + A:] = 0
    return dict(wf=rn(ks, Q, R, scale=0.5), bf=rn(R, scale=0.1), W1=W1, b1=rn(L, 2 * R, scale=0.1),
                W2=rn(L, R + S, R, scale=1.0 / R ** 0.5), b2=rn(L, R + S, scale=0.1),
                Wp1=rn(S, S, scale=1.5 / S ** 0.5), bp1=rn(S, scale=0.1), Wp2=rn(Q, S, scale=2.0 / S ** 0.5),
                bp2=rn(Q, scale=0.1), up_w=rn(U) if U else None, up_b=rn(1, scale=0.1) if U else None,
                dil=list(dil), ks=ks, U=U, n_pad=3)


def _bf(x):
    return x.to(torch.bfloat16).to(F32)


def _libm(fn, x, g):
    """fn(x) in float32 within 2 ulp: the correctly rounded value moved by -1, 0 or +1 ulp"""
    y = fn(x.double()).float()
    k = torch.randint(-1, 2, y.shape, generator=g, dtype=torch.int32)
    moved = (y.view(torch.int32) + k).view(F32)
    return torch.where(y == 0, y, moved)


def _acc(a, w, g):
    """a (B, K) @ w (N, K)^T with bf16 operands, as k16 tensor-core steps in K order: each step adds 16 exact products
    to the fp32 accumulator and rounds once, to nearest or toward zero at random"""
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64)
    for k0 in range(0, a.shape[1], 16):
        s = acc + a[:, k0:k0 + 16].double() @ w[:, k0:k0 + 16].double().t()
        rn = s.float()
        tz = torch.where(rn.double().abs() > s.abs(), torch.nextafter(rn, torch.zeros_like(rn)), rn)
        acc = torch.where(torch.rand(rn.shape, generator=g) < 0.5, rn, tz).double()
    return acc.float()


def emulate(pk, B, T, h, fault=None, seed=1):
    """positions 0 .. T-1 from a one-sample seed: (codes (B, T + 1), q [L x (B, T, R)], logits (B, T, Q))"""
    g = torch.Generator().manual_seed(seed)
    ks, U, n_pad, dil = pk["ks"], pk["U"], pk["n_pad"], pk["dil"]
    L, R2, _ = pk["W1"].shape
    R, Q, A, Th = R2 // 2, pk["wf"].shape[1], h.shape[1], h.shape[2]
    Ap = pk["W1"].shape[2] - ks * R
    Ak = (Ap + 63) // 64 * 64
    # the kernel's K order: [aux (Ak) | taps | x(t)]
    W1 = [_bf(torch.cat([torch.nn.functional.pad(pk["W1"][l][:, ks * R:], (0, Ak - Ap)), pk["W1"][l][:, :ks * R]], 1))
          for l in range(L)]
    W2 = [_bf(pk["W2"][l]) for l in range(L)]
    Wp1, Wp2 = _bf(pk["Wp1"]), _bf(pk["Wp2"])
    codes = torch.full((B, T + 1), Q // 2, dtype=torch.long)
    codes[:, 0] = torch.randint(0, Q, (B,), generator=g)
    q = [torch.zeros(B, T, R, dtype=F32) for _ in range(L)]
    logits = torch.zeros(B, T, Q, dtype=F32)
    for t in range(T):
        x = pk["bf"][None].expand(B, R).clone()
        for k in range(ks):
            pp = t - (ks - 1 - k)
            if pp >= 0:
                x = x + pk["wf"][k][codes[:, pp] % Q]
        j = max(t - n_pad, 0) + (1 if fault == "aux" else 0)
        if U:
            hv = h[:, :, min(j // U, Th - 1)]
            aux = _bf(DL.fma32(hv, pk["up_w"][j % U].expand_as(hv), pk["up_b"].expand_as(hv)))
        else:
            aux = _bf(h[:, :, min(j, Th - 1)])
        aux = torch.nn.functional.pad(aux, (0, Ak - A))
        skip = None
        for l in range(L):
            xb = _bf(x)
            q[l][:, t] = xb
            taps = []
            for jj in range(ks - 1):
                p = t - (ks - 1 - jj) * dil[l]
                if fault == "tap" and l == 1 and jj == 0:
                    p += 1                                          # the neighbouring slot
                if p >= 0:
                    taps.append(q[l][:, p])
                else:
                    taps.append(torch.full_like(xb, 0.25 if fault == "pre_start" else 0.0))
            pre = _acc(torch.cat([aux] + taps + [xb], 1), W1[l], g) + pk["b1"][l]
            s = 1.0 / (1.0 + _libm(torch.exp, -pre[:, :R], g))
            z = _bf(s * _libm(torch.tanh, pre[:, R:], g))
            d = _acc(z, W2[l], g)
            x = x + (d[:, :R] + pk["b2"][l][:R])
            if fault == "x" and l == 1 and t == T // 2:
                x[0, 3] = x[0, 3] + 3 * 2.0 ** (torch.frexp(x[0, 3])[1] - 8)    # three bf16 ulps
            v = d[:, R:] + (0 if fault == "skip_bias" and l == 2 else pk["b2"][l][R:])
            skip = v if l == 0 else skip + v
        r1 = _bf(torch.relu(_acc(_bf(torch.relu(skip)), Wp1, g) + pk["bp1"]))
        lg = _acc(r1, Wp2, g) + pk["bp2"]
        logits[:, t] = lg
        if t % 2:
            codes[:, t + 1] = lg.argmax(1)
        else:
            codes[:, t + 1] = torch.multinomial(torch.softmax(lg.double(), 1), 1, generator=g)[:, 0]
    return codes, q, logits


def _aux(pk, B, T, A=5, seed=2):
    U = pk["U"]
    frames = (T + U - 1) // U + 1 if U else T + 1
    return torch.randn(B, A, frames, generator=torch.Generator().manual_seed(seed)).to(F32)


def _check(pk, codes, q, logits, T):
    h = pk["_h"]
    return DL.check_window(pk, codes, h, q, [0] * len(q), 0, T, logits)


@pytest.mark.parametrize("ks,U", [(2, 0), (2, 4), (3, 0), (3, 5)])
def test_checker_accepts_the_emulation(ks, U):
    pk = _model(ks, U, seed=10 * ks + U)
    B, T = 3, 256
    pk["_h"] = _aux(pk, B, T)
    codes, q, logits = emulate(pk, B, T, pk["_h"], seed=ks + U)
    rep = _check(pk, codes, q, logits, T)
    print("ks %d U %d: %s" % (ks, U, rep))
    assert rep["queue"] <= 1.0 and rep["logits"] <= 1.0


def test_checker_accepts_the_emulation_at_recipe_width():
    pk = _model(3, 4, R=256, S=256, Q=256, seed=5)
    B, T = 2, 48
    pk["_h"] = _aux(pk, B, T)
    codes, q, logits = emulate(pk, B, T, pk["_h"], seed=6)
    rep = _check(pk, codes, q, logits, T)
    print("R 256: %s" % rep)
    assert rep["queue"] <= 1.0 and rep["logits"] <= 1.0


FAULTS = {
    "tap": r"layer 1 -> 2 residual",                        # a tap read from the neighbouring slot (layer 1, d = 2)
    "aux": r"layer 0 -> 1 residual",                        # aux one sample late
    "x": r"layer 1 -> 2 residual: position 32, utterance 0 .*channel 3:",   # one channel of x_2 three bf16 ulps off
    "skip_bias": r"^logits",                                # layer 2's skip bias dropped
    "pre_start": r"layer 0 -> 1 residual: position [01],",  # a tap before position 0 that is not zero
}


@pytest.mark.parametrize("R", [16, 256])
@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_rejects_planted_fault(fault, R):
    pk = _model(3, 4, R=R, S=R, seed=7)
    B, T = 2, 64
    pk["_h"] = _aux(pk, B, T)
    codes, q, logits = emulate(pk, B, T, pk["_h"], fault=fault, seed=3)
    with pytest.raises(AssertionError) as ei:
        _check(pk, codes, q, logits, T)
    print(fault, R, str(ei.value))
    assert re.search(FAULTS[fault], str(ei.value)), str(ei.value)


def _fma_exact(a, b, c):
    """the correctly rounded float32 of a * b + c, from exact rationals"""
    out = []
    for x, y, z in zip(a.tolist(), b.tolist(), c.tolist()):
        e = fractions.Fraction(x) * fractions.Fraction(y) + fractions.Fraction(z)
        lo = np.float32(float(e))                    # within one float32 step of e; pick the nearest, ties to even
        cands = sorted({np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))},
                       key=lambda v: (abs(fractions.Fraction(float(v)) - e),
                                      int(np.array(v, np.float32).view(np.uint32)) & 1))
        out.append(cands[0])
    return torch.tensor(np.array(out, np.float32))


def test_fma32_is_correctly_rounded():
    a = torch.tensor([1 + 2 ** -12] * 3, dtype=F32)
    c = torch.tensor([2.0 ** -80, -2.0 ** -80, 0.0], dtype=F32)
    # a * a = 1 + 2^-11 + 2^-24 is a float32 midpoint; the float64 add loses c, so only TwoSum knows the side
    got = DL.fma32(a, a, c)
    assert got.tolist() == [1 + 2 ** -11 + 2 ** -23, 1 + 2 ** -11, 1 + 2 ** -11]
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(4000, generator=g), torch.randn(4000, generator=g)
    c = torch.randn(4000, generator=g) * torch.exp2(torch.randint(-40, 10, (4000,), generator=g).float())
    assert torch.equal(DL.fma32(a, b, c), _fma_exact(a, b, c))


def test_bf16_neighbours():
    q = torch.tensor([1.0, -1.0, 0.0, 1.5, 2.0 ** -133, 3.0], dtype=torch.float64)
    hd, hu = DL.bf16_halfgaps(q)
    assert hd.tolist() == [2.0 ** -9, 2.0 ** -8, 2.0 ** -134, 2.0 ** -8, 2.0 ** -134, 2.0 ** -7]
    assert hu.tolist() == [2.0 ** -8, 2.0 ** -9, 2.0 ** -134, 2.0 ** -8, 2.0 ** -134, 2.0 ** -7]
    # a value known to within e: exact where no rounding boundary is inside [v - e, v + e], else the midpoint of the
    # two possible roundings and half their distance
    r, gap, st = DL.round_interval(torch.tensor([1.0 + 2.0 ** -8, 1.0 + 2.0 ** -10], dtype=torch.float64),
                                   torch.tensor([2.0 ** -20, 2.0 ** -20], dtype=torch.float64))
    assert st.tolist() == [True, False] and gap.tolist() == [2.0 ** -8, 0.0] and r.tolist() == [1.0 + 2.0 ** -8, 1.0]
