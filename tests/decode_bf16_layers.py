# -*- coding: utf-8 -*-
"""Layer-by-layer float64 check of the bf16 decoder (csrc/decode_bf16.cu), teacher-forced from its own dilation queues.

Plain torch in float64 on whatever device the inputs live on.  The decoder keeps, per layer l, a queue of bf16(x_l(t)),
the layer's input at position t, written in the res epilogue from the same registers and with the same ``cvt`` that
fill the gate's A operand; ``logits_out`` holds each step's fp32 logits.  ``check_window`` takes those observations over
a window of positions and checks every stage of every layer at every position and row from the kernel's own operands.

Accumulation bound (``mma_product``).  bf16 x bf16 products are exact in fp32.  A wgmma k16 instruction adds 16
products to the fp32 accumulator, at worst as two steps of 8 products each.  In one step the 9 addends (8 products and
the accumulator) are aligned to the largest exponent and summed, and the sum is rounded to fp32 (not necessarily to
nearest).  Each addend then loses less than 2^-23 M and the rounding less than 2^-23 M, where M is the largest of |the
accumulator before|, |after| and the largest product of the step: at most 20 * 2^-23 M per k16 step, times C_ACC = 2
for the same reasons ``tc_reference.lin_bound`` carries it.  Summed over the K / 16 steps in the kernel's K order, with
M taken from the exact partial sums (plus the input error and a factor 1 + 2 C G for the error the partial sums have
already picked up):
    e_acc = C sum_g max(|S_g-1|, |S_g|, max_k in g |a_k w_k|) (1 + 2 C G) + |w| e_in,   C = C_ACC 20 2^-23,
over the G = K / 16 steps g (S_g the exact partial sum after step g).
This is lin_bound's model applied per hardware step: lin_bound charges one unit per term against sum |a||w| (about
2 K 2^-23 sum |a||w|), which at K = ks R + Ak ~ 1 000 exceeds a bf16 step of z for most z; the partial sums of a gate
row grow like the square root of K, so this bound is smaller by about that factor.

Stages and bounds (u = 2^-24):
* Front.  x_0 = bf + wf[0][q_0] + wf[1][q_1] (+ wf[2][q_2]) added in fp32 in that order (missing history adds
  nothing), restated in float32 in the same order.  Layer 0's queue must equal its bf16 rounding exactly.
* Aux.  bf16_rn(fmaf(h[tf][a], up_w[j % U], up_b)) with j = max(t - n_pad, 0), tf = min(j // U, last frame); bf16_rn(h)
  for U = 0; zero for a >= A.  ``fma32`` computes the fused multiply-add exactly: the float64 product is exact, TwoSum
  gives the rounding error of the float64 add, and an fp32 midpoint with a nonzero error is rounded toward that error.
* Gate of layer l.  Operands: the observed q_l(t - (ks-1-j) d_l) (zero before position 0), q_l(t) and the aux; weights
  ``to_bf16`` of the fp32 parameters (the rounding of ``_decode_bf16_pack``), in the kernel's K order [aux (Ak) | taps
  j = 0 .. ks-2 | x(t)].  The pre-activation bound is e_acc plus u (|acc| + |b1|) for the bias add; the gate model is ``GATE_LIBM``
  (``sigmoidf_`` = 1 / (1 + expf(-x)) and ``tanhf``), z = s th with e_z = |th| e_s + s e_th + e_s e_th + 2u |z|.
* bf16 roundings of a value known to within e (z, relu(skip sum), relu(post-1)).  The kernel's operand lies between
  rn(v - e) and rn(v + e) (rounding is monotone).  Where that is one value it is exact; where [v - e, v + e] straddles a
  rounding boundary the reference takes the midpoint of the two and carries half their distance downstream as an input
  error through |W|.  Where one such operand dominates an element's bound, that element's err/bound can come close
  to 1 in a correct kernel.
* Residual stream.  The fp32 x_l is never observed, only bf16(x_l), so it is carried as an interval [lo, hi]: exact for
  x_0; each layer adds d + b2 with two fp32 roundings, so x_{l+1} lies in [lo + r - E, hi + r + E] with r the float64
  d + b2, e_d its product bound (e_acc, with the input error of z through |W2|) and E = e_d + u (max(|lo|, |hi|) +
  3 (|r| + e_d)) (+ 2^-50 of the same for the float64 arithmetic).  That interval is intersected with the preimage of
  the observed q_{l+1} under round to nearest even, [q - h_down, q + h_up] (half the distance to each bf16 neighbour).
  The intersection resets the interval at every layer, so it does not grow with depth; its width is one bf16 ulp of
  x_l plus 2E.  At the recipe sizes E is the larger term: 12-27 % of the z intervals still straddle a bf16 boundary,
  and their half steps pass into E through |W2| (``width`` in the report).
* Skip and post network.  skip = sum_l (W2skip z + b2skip) added in layer order from l = 0 (each term one rounding, each
  partial sum one more); relu -> bf16 (straddle as above); post-1 + bp1 -> relu -> bf16; post-2 + bp2, compared with
  ``logits_out`` element by element (``tc_reference.assert_within``; its column group of 32 is the owning CTA).

Ratios reported (the largest over the window, every row and channel):
* ``queue``: for layers 1 .. L-1, the distance from the observed bf16 value q to the predicted interval, divided by
  half the distance from q to its bf16 neighbour on that side.  It is 0 when q lies inside the interval and exceeds 1
  exactly when the interval and the preimage of q do not meet, which fails.  A correct kernel spreads it over [0, 1]:
  it measures where x fell between two bf16 values, not a margin.
* ``width``: the widest predicted interval before the intersection, in bf16 ulps at the magnitude max(|x_l|, |q|):
  how sharp the queue check is.  (Where x_l and d cancel, q is far smaller than x_l and the interval spans many of
  q's own ulps; the check there is as sharp as x_l's rounding allows.)
* ``logits``: |logit - ref| / bound.
* ``straddles``: bf16 roundings whose input interval holds more than one bf16 value; ``z_straddle_frac`` the largest
  fraction of one layer's z values that do.
The front is exact or fails, so it has no ratio.
"""
import torch

from tests import tc_reference as ref
from tests.test_bf16_host import to_bf16

F64 = torch.float64
U = ref.U


def fma32(a, b, c):
    """float32 tensor of the correctly rounded a * b + c (fmaf) of float32 tensors"""
    p = a.to(F64) * b.to(F64)                       # exact: 24 + 24 significant bits
    c = c.to(F64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                 # TwoSum: p + c = s + err exactly
    r = s.to(torch.float32)
    r64 = r.to(F64)
    inf = torch.full_like(r, float("inf"))
    other = torch.nextafter(r, torch.where(s > r64, inf, -inf)).to(F64)
    mid = (s != r64) & ((s - r64) * 2 == (other - r64))
    nudged = torch.nextafter(s, torch.where(err > 0, inf.to(F64), -inf.to(F64))).to(torch.float32)
    return torch.where(mid & (err != 0), nudged, r)


def bf16_rn(x):
    """float64 tensor of the bf16 rounding of x (via fp32: x already an fp32 value, or a reference value)"""
    return to_bf16(x.to(torch.float32))


def bf16_halfgaps(q):
    """(h_down, h_up): half the distance from bf16 values q (float64) to their lower and upper bf16 neighbours"""
    b = q.to(torch.float32).to(torch.bfloat16)
    bits = b.view(torch.int16).to(torch.int32)     # sign and magnitude: +1 is one step away from zero for either sign
    zero = (bits & 0x7FFF) == 0

    def val(bi):
        return bi.to(torch.int16).view(torch.bfloat16).to(F64)
    qv = b.to(F64)
    away, toward = (val(bits + 1) - qv).abs(), (qv - val(bits - 1)).abs()
    tiny = 2.0 ** -133                             # the smallest bf16 subnormal
    toward = torch.where(zero, torch.full_like(toward, tiny), toward)
    pos = bits >= 0
    h_up = torch.where(pos, away, toward) / 2
    h_down = torch.where(pos, toward, away) / 2
    return h_down, h_up


def _round_between(lo, hi):
    """(midpoint, half span, straddle mask) of the bf16 roundings rn(lo) .. rn(hi)"""
    rl, rh = bf16_rn(lo), bf16_rn(hi)
    return (rl + rh) / 2, (rh - rl) / 2, rh != rl


def round_interval(v, e):
    """bf16 operand of a value known to within e: the kernel's operand lies in [rn(v - e), rn(v + e)]; returns its
    midpoint, half its span (0 unless a rounding boundary lies inside [v - e, v + e]) and the straddle mask"""
    return _round_between(v - e, v + e)


def _relu_round(v, e):
    """relu -> bf16 of a value known to within e (relu is monotone)"""
    return _round_between((v - e).clamp_min(0), (v + e).clamp_min(0))


STEP = 16                                  # K of one wgmma instruction
C_STEP = ref.C_ACC * 20 * 2.0 ** -23       # per k16 step: two 8-term steps of 9 addends and one rounding each


def mma_product(a, ea, w):
    """a (..., K) in the kernel's K order, known to within ea (a tensor like a, or 0), times bf16 w (N, K)^T, accumulated
    by k16 wgmma steps in K order: (exact product of a and w, bound).  See the module docstring."""
    K = a.shape[-1]
    G = -(-K // STEP)
    assert C_STEP * G < 0.5
    pad = G * STEP - K
    ea = torch.zeros_like(a) + ea
    if pad:
        a, ea, w = (torch.nn.functional.pad(t, (0, pad)) for t in (a, ea, w))
    ac = a.reshape(*a.shape[:-1], G, STEP)
    wc = w.reshape(w.shape[0], G, STEP)
    step = torch.einsum("...gk,ngk->...ng", ac, wc)
    S = step.cumsum(-1)                                                  # partial sums after each step
    amax = (ac.abs() + ea.reshape(ac.shape)).amax(-1)                    # (..., G)
    tmax = amax[..., None, :] * wc.abs().amax(-1)                         # (..., N, G): the largest product of a step
    e_in = ea @ w.abs().t()                                               # the input error through |w|
    M = torch.maximum(torch.maximum((S - step).abs(), S.abs()), tmax) + e_in[..., None]
    return S[..., -1], C_STEP * M.sum(-1) * (1 + 2 * C_STEP * G) + e_in


def _linear(a, ea, w, b):
    """mma_product plus the bias b in one fp32 add"""
    acc, e = mma_product(a, ea, w)
    return acc + b, e + U * (acc.abs() + e + b.abs())


class LayerCheckError(AssertionError):
    pass


def _where(R, bc, b, c):
    cl, row = (b // bc, b % bc) if bc else (0, b)
    return "utterance %d (cluster %d row %d), channel %d: CTA slice %d, 64-channel tile %d" % (
        b, cl, row, c, c // (R // 8), c // 64)


def check_window(pk, codes, h, q, q_first, t0, t1, logits, bc=None):
    """Check positions t0 .. t1 - 1 of every row.

    pk: dict of the model in ``WaveNet._pack`` layout (fp32): wf (ks, Q, R), bf (R), W1 (L, 2R, ks R + Ap), b1 (L, 2R),
        W2 (L, R + S, R), b2 (L, R + S), Wp1 (S, S), bp1 (S), Wp2 (Q, S), bp2 (Q), up_w (U) / up_b (1) or None, and the
        ints / lists dil, ks, U, n_pad.
    codes: (B, >= t1) int, the codes the front embedding reads at each position.  h: (B, A, Th) fp32 aux frames.
    q: list of L tensors (B, T_l, R), the observed bf16(x_l) at positions q_first[l] .. (any float dtype).
    logits: (B, t1 - t0, Q) fp32 ``logits_out``, NaN where the kernel wrote none.  bc: rows per cluster (messages).
    Returns the report of the module docstring; raises LayerCheckError / AssertionError naming the failing spot."""
    dev = h.device
    ks, Uf, n_pad, dil = pk["ks"], pk["U"], pk["n_pad"], list(pk["dil"])
    wf, bf = pk["wf"].float(), pk["bf"].float()
    W1, W2 = pk["W1"], pk["W2"]
    L, R2, K1 = W1.shape
    R = R2 // 2
    S = W2.shape[1] - R
    Q = wf.shape[1]
    Ap = K1 - ks * R
    Ak = (Ap + 63) // 64 * 64
    B, A, Th = h.shape
    T = t1 - t0
    pos = torch.arange(t0, t1, device=dev)
    codes = torch.as_tensor(codes, device=dev).long()
    rep = {"queue": 0.0, "width": 0.0, "logits": 0.0, "straddles": 0, "z_straddle_frac": 0.0}

    def getq(l, p):
        """observed q_l at positions p (T,) for every row: (B, T, R) float64, zero before position 0"""
        idx = p - q_first[l]
        ok = p >= 0
        assert bool((idx[ok] >= 0).all()) and bool((idx < q[l].shape[1]).all()), ("queue history too short", l)
        v = q[l][:, idx.clamp_min(0)].to(F64)
        return torch.where(ok[None, :, None], v, torch.zeros_like(v))

    # ---- front: x_0 in fp32, tap order ----
    x0 = bf[None, None, :].expand(B, T, R).clone()
    for k in range(ks):
        pp = pos - (ks - 1 - k)
        cq = codes[:, pp.clamp_min(0)] % Q                                     # (B, T)
        add = wf[k][cq]                                                         # (B, T, R)
        x0 = torch.where((pp >= 0)[None, :, None], x0 + add, x0)
    q0 = getq(0, pos)
    bad = bf16_rn(x0) != q0
    if bool(bad.any()):
        b, t, c = (int(v) for v in torch.nonzero(bad)[0])
        raise LayerCheckError("front: layer 0 queue differs from bf16(x_0) at position %d, %s: got %.9g, want %.9g "
                              "(%d values differ)" % (t0 + t, _where(R, bc, b, c), float(q0[b, t, c]),
                                                      float(bf16_rn(x0)[b, t, c]), int(bad.sum())))

    # ---- aux operand (B, T, Ap) ----
    j = (pos - n_pad).clamp_min(0)
    if Uf > 0:
        tf = (j // Uf).clamp_max(Th - 1)
        hv = h[:, :, tf].float()                                                # (B, A, T)
        uw = pk["up_w"].float()[j % Uf][None, None, :].expand_as(hv)
        ub = pk["up_b"].float().reshape(1, 1, 1).expand_as(hv)
        av = fma32(hv, uw, ub)
    else:
        av = h[:, :, j.clamp_max(Th - 1)].float()
    aux = torch.zeros(B, T, Ak, dtype=F64, device=dev)                        # zero past A and in the Ak padding
    aux[:, :, :A] = bf16_rn(av.transpose(1, 2))

    # ---- layers ----
    lo = hi = x0.to(F64)
    skip, e_skip = 0, 0
    for l in range(L):
        d = dil[l]
        # the kernel's K order: [aux (Ak) | taps j = 0 .. ks-2 | x(t)]
        a = torch.cat([aux] + [getq(l, pos - (ks - 1 - jj) * d) for jj in range(ks - 1)] + [getq(l, pos)], -1)
        w1 = to_bf16(torch.cat([torch.nn.functional.pad(W1[l][:, ks * R:], (0, Ak - Ap)), W1[l][:, :ks * R]], 1))
        pre, e_pre = _linear(a, 0, w1, pk["b1"][l].to(F64))
        s, th, es, eth = ref._gate_parts(pre, e_pre, ref.GATE_LIBM)
        z = s * th
        ez = th.abs() * es + s * eth + es * eth + 2 * U * z.abs()
        zb, ezb, st = round_interval(z, ez)
        rep["straddles"] += int(st.sum())
        rep["z_straddle_frac"] = max(rep["z_straddle_frac"], float(st.double().mean()))
        w2 = to_bf16(W2[l])
        b2 = pk["b2"][l].to(F64)
        dv, ed = mma_product(zb, ezb, w2)                # biases added below, with their own roundings
        # residual: x_{l+1} = fl(x_l + fl(d + b2))
        r = dv[..., :R] + b2[:R]
        tm = r.abs() + ed[..., :R]
        xm = torch.maximum(lo.abs(), hi.abs())
        E = ed[..., :R] + U * (xm + 3 * tm) + 2.0 ** -50 * (xm + tm)
        lo, hi = lo + r - E, hi + r + E
        if l + 1 < L:
            qv = getq(l + 1, pos)
            hd, hu = bf16_halfgaps(qv)
            below = (qv - hi).clamp_min(0) / hd           # q above the interval: distance down to it
            above = (lo - qv).clamp_min(0) / hu           # q below the interval
            ratio = torch.maximum(below, above)
            ulp = torch.ldexp(torch.ones_like(xm), torch.frexp(torch.maximum(xm, qv.abs()))[1] - 8)
            width = (hi - lo) / ulp
            rep["width"] = max(rep["width"], float(width.max()))
            worst = float(ratio.max())
            if not worst <= 1.0:
                i = int(torch.argmax(ratio.reshape(-1)))
                b, t, c = (int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
                raise LayerCheckError(
                    "layer %d -> %d residual: position %d, %s: observed bf16(x_%d) %.9g outside the predicted "
                    "[%.9g, %.9g] (err/bound %.3g; %d values fail)" % (
                        l, l + 1, t0 + t, _where(R, bc, b, c), l + 1, float(qv[b, t, c]), float(lo[b, t, c]),
                        float(hi[b, t, c]), worst, int((ratio > 1).sum())))
            rep["queue"] = max(rep["queue"], worst)
            lo, hi = torch.maximum(lo, qv - hd), torch.minimum(hi, qv + hu)
        # skip: v = fl(d + b2skip); skip = v, then fl(skip + v)
        v = dv[..., R:] + b2[R:]
        ev = ed[..., R:] + U * (v.abs() + ed[..., R:])
        if l == 0:
            skip, e_skip = v, ev
        else:
            skip = skip + v
            e_skip = e_skip + ev + U * (skip.abs() + e_skip + ev)

    # ---- post network ----
    rs, ers, st = _relu_round(skip, e_skip)
    rep["straddles"] += int(st.sum())
    p1, ep1 = _linear(rs, ers, to_bf16(pk["Wp1"]), pk["bp1"].to(F64))
    r1, er1, st = _relu_round(p1, ep1)
    rep["straddles"] += int(st.sum())
    lg, elg = _linear(r1, er1, to_bf16(pk["Wp2"]), pk["bp2"].to(F64))
    got = torch.as_tensor(logits, device=dev).to(F64)
    seen = ~torch.isnan(got)
    assert bool(seen.any()), "no logits observed"
    got = torch.where(seen, got, lg)
    rep["logits"] = ref.assert_within(got, lg, elg, "logits (b = utterance, t = position - %d, column group = CTA)" % t0)
    return rep
