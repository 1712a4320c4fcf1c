# -*- coding: utf-8 -*-
"""float64 reference of every tensor-core stage of the tf32 training path, with an element-wise error bound per stage.

Plain torch in float64 on whatever device the inputs live on (the GPU tests pass device tensors, the CPU tier CPU
ones).  Every function works on the packed layouts of ``include/wnb200.h`` (channels-last activations (B, T, C),
W1 (2R, K1) with K1 = ks*R + Ap, W2res (R, R), Wskip (S, L*R), wp1 (S, S), wp2 (Q, S)) and returns ``(ref, bound)``:
the exact result of the stage for the kernel's own fp32 inputs, and a bound on |kernel - ref| per element.

Error model
-----------
tf32 operands.  wgmma reads the raw fp32 bit patterns of both operands as tf32 (no ``cvt`` is issued anywhere): the
low 13 mantissa bits are dropped (``TF32_RULE = "truncate"``, measured by ``tests/test_gpu_tc_exact.py``).  The
reference converts its operands with ``to_tf32`` the same way, so every product of two tf32 numbers (11 x 11
significant bits) is exact in fp32 and in fp64: the only rounding left in a contraction is fp32 accumulation.

Linear stages.  A sum of K exact products accumulated in fp32 in any order satisfies
|fl(sum) - sum| <= gamma_K * sum |terms| with gamma_K ~ K * 2^-24 (Higham, Accuracy and Stability, 3.1).  The bound
used is  C_ACC * K * 2^-23 * (|A^| |B^|)_ij  with C_ACC = 2, i.e. four times gamma_K: the tensor cores align the
addends of an 8-term dot product to the largest exponent and need not round to nearest, which costs up to one more
unit per addition.  Epilogue operations (bias, residual, the split-K slot reduce, += into the caller's buffer) each add
one fp32 rounding, 2^-24 times the magnitude of their operands.

Gate stages.  The pre-activations a (sigmoid branch) and g (tanh branch) carry the linear bounds e_a, e_g.  The kernel
evaluates tanh with ``tanh.approx.f32`` (relative error <= 2^-10.987, PTX ISA) and sigmoid as 0.5*tanh(0.5 a) + 0.5,
so with s = sigmoid(a), th = tanh(g):
    e_s  <= s(1-s) e_a + 0.1 e_a^2 + |s - 1/2| eps + 2u           (|sigmoid''| <= 0.1)
    e_th <= (1-th^2) e_g + 0.77 e_g^2 + |th| eps + u              (|tanh''|  <= 0.77)
    z = s th:                  e_z  <= |th| e_s + s e_th + e_s e_th + 2u |z|
    da = dz th s(1-s):         e_da <= |th| s(1-s) e_dz + |dz| (s(1-s) e_th + |th| |1-2s| e_s + |th| e_s^2)
                                       + e_dz (e_s + e_th) + 6u |dz th s(1-s)|
    dg = dz s (1-th^2):        e_dg <= s(1-th^2) e_dz + |dz| ((1-th^2) e_s + 2 s |th| e_th + s e_th^2)
                                       + e_dz (e_s + e_th) + 6u |dz| s
first order in the propagated errors plus the second-order terms above (eps = 2^-10.987, u = 2^-24).

fp32 (SIMT) path.  ``math_mode="fp32"`` multiplies fp32 operands as given (``cv=exact``: every product is exact in
float64) and accumulates with one ``fmaf`` per term, so the linear bound above holds with room to spare (gamma_K is
K * 2^-24 for any order).  Its gates are ``sigmoidf_(a) = 1 / (1 + expf(-a))`` with IEEE division and libm ``tanhf``;
without fast-math both ``expf`` and ``tanhf`` are within 2 ulp (CUDA C Programming Guide, mathematical functions), i.e.
relative error <= LIBM_REL = 2^-22.  With e = exp(-a), 1 - s = e / (1 + e):
    s^ = s (1 + d3) / ((1 + d2)(1 + (1-s) d1)),  |d1| <= LIBM_REL, |d2|, |d3| <= u
so  e_s <= s(1-s) e_a + 0.1 e_a^2 + s ((1-s) LIBM_REL + 3u)  (3u: two roundings plus the second-order terms, valid
while expf(-a) does not overflow, |a| < 88), and  e_th <= (1-th^2) e_g + 0.77 e_g^2 + |th| LIBM_REL.  ``gate_fn``
selects the model: GATE_TANH_APPROX (the tensor-core kernels, the default) or GATE_LIBM (the SIMT kernels).

Stages whose input never leaves the chip (the fused per-block forward keeps z in shared memory) take the propagated
bound of that input as ``e_in``: the kernel's operand then differs from the reference's by e_in plus one tf32
conversion step of each (2^-10 relative each), which enters through |W|.
"""
import numpy as np
import torch

TF32_RULE = "truncate"          # how the tensor cores read an fp32 operand; "truncate" or "round" (to nearest)
C_ACC = 2.0
U = 2.0 ** -24                  # fp32 unit roundoff
TANH_REL = 2.0 ** -10.987       # tanh.approx.f32
TF32_REL = 2.0 ** -10           # largest relative change of one tf32 conversion (truncation)
LIBM_REL = 2.0 ** -22           # expf / tanhf without fast-math: 2 ulp
F64 = torch.float64


def GATE_TANH_APPROX(s, th):
    """function error of the tensor-core gates: (e_s, e_th) of sigmoid = 0.5 tanh.approx(a/2) + 0.5, tanh.approx"""
    return (s - 0.5).abs() * TANH_REL + 2 * U, th.abs() * TANH_REL + U


def GATE_LIBM(s, th):
    """function error of the SIMT gates: (e_s, e_th) of 1 / (1 + expf(-a)) and tanhf"""
    return s * ((1 - s) * LIBM_REL + 3 * U), th.abs() * LIBM_REL


# ------------------------------------------------------------------------------------------------------------------
# operand conversion and helpers
# ------------------------------------------------------------------------------------------------------------------
def to_tf32(x, rule=None):
    """fp32 tensor -> float64 tensor of the tf32 value the tensor cores multiply with."""
    rule = TF32_RULE if rule is None else rule
    b = x.detach().to(torch.float32).contiguous().view(torch.int32)
    if rule == "round":
        b = b + 0x1000           # round half away from zero on the magnitude (carries into the exponent correctly)
    elif rule != "truncate":
        raise ValueError(rule)
    return (b & ~0x1FFF).view(torch.float32).to(F64)


def exact(x):
    """no conversion (the composed fp64 model of the CPU tier)"""
    return x.detach().to(F64)


def tshift(x, s):
    """y[:, t] = x[:, t + s] (zero outside [0, T)) on (B, T, C) -- the TMA zero fill of a shifted box."""
    T = x.shape[1]
    y = torch.zeros_like(x)
    if s >= 0:
        if s < T:
            y[:, :T - s] = x[:, s:]
    elif -s < T:
        y[:, -s:] = x[:, :T + s]
    return y


def _mm(a, w, cv):
    """a (..., K) times w (N, K)^T with converted operands: (sum, sum of |terms|)"""
    a, w = cv(a), cv(w)
    return a @ w.t(), a.abs() @ w.abs().t()


def lin_bound(mag, K):
    """accumulation bound of K fp32-accumulated exact products whose absolute values sum to `mag`"""
    return C_ACC * K * 2.0 ** -23 * mag


def taps(x, ks, d):
    """the ks dilated taps of a causal conv, oldest first: x(t - (ks-1-j) d)"""
    return [tshift(x, -(ks - 1 - j) * d) for j in range(ks)]


# ------------------------------------------------------------------------------------------------------------------
# forward stages
# ------------------------------------------------------------------------------------------------------------------
def gate_pre(xin, haux, w1, b1, d, ks, cv=to_tf32):
    """pre-activations (B,T,2R) = sum_j x(t-(ks-1-j)d) W1[:, tap j]^T + aux W1[:, aux]^T + b1, and their bound"""
    R = xin.shape[-1]
    K1 = w1.shape[1]
    acc = 0
    mag = 0
    for j, xj in enumerate(taps(xin, ks, d)):
        v, m = _mm(xj, w1[:, j * R:(j + 1) * R], cv)
        acc, mag = acc + v, mag + m
    v, m = _mm(haux, w1[:, ks * R:], cv)
    acc, mag = acc + v, mag + m
    b = b1.to(F64)
    pre = acc + b
    return pre, lin_bound(mag, K1) + U * (acc.abs() + b.abs())


def _gate_parts(pre, e_pre, gate_fn):
    R = pre.shape[-1] // 2
    a, g, ea, eg = pre[..., :R], pre[..., R:], e_pre[..., :R], e_pre[..., R:]
    s, th = torch.sigmoid(a), torch.tanh(g)
    fs, fth = gate_fn(s, th)
    es = s * (1 - s) * ea + 0.1 * ea * ea + fs
    eth = (1 - th * th) * eg + 0.77 * eg * eg + fth
    return s, th, es, eth


def gate_fwd(xin, haux, w1, b1, d, ks, cv=to_tf32, gate_fn=GATE_TANH_APPROX):
    """z = sigmoid(a) tanh(g) (B,T,R) and its bound"""
    pre, e = gate_pre(xin, haux, w1, b1, d, ks, cv)
    s, th, es, eth = _gate_parts(pre, e, gate_fn)
    z = s * th
    return z, th.abs() * es + s * eth + es * eth + 2 * U * z.abs()


def _in_term(x, e_in, w):
    """contribution of an on-chip operand known only to within e_in: |W| (e_in + two tf32 steps)"""
    if e_in is None:
        return 0
    xa = x.to(F64).abs()
    return (e_in + TF32_REL * (2 * xa + e_in)) @ w.to(F64).abs().t()


def res_out(xin, z, w2res, b2res, e_z=None, cv=to_tf32):
    """xout = xin + z W2res^T + b2res (the residual output of a block)"""
    acc, mag = _mm(z, w2res, cv)
    b, x = b2res.to(F64), xin.to(F64)
    out = acc + b + x
    return out, (lin_bound(mag, z.shape[-1]) + _in_term(z, e_z, w2res)
                 + 2 * U * (acc.abs() + b.abs() + x.abs()))


def skip_gemm(zall, wskip, bskip, relu, e_z=None, cv=to_tf32, skip_in=None):
    """skip = zall Wskip^T + bskip [+ skip_in, the per-block accumulation], optionally rectified"""
    acc, mag = _mm(zall, wskip, cv)
    b = 0 if bskip is None else bskip.to(F64)
    out = acc + b
    bound = lin_bound(mag, zall.shape[-1]) + _in_term(zall, e_z, wskip) + U * (acc.abs() + abs(b))
    if skip_in is not None:
        si = skip_in.to(F64)
        out = out + si
        bound = bound + U * (out.abs() + si.abs())
    if relu:
        out = out.clamp_min(0)
    return out, bound


def post_fwd(skip_r, wp1, bp1, wp2, bp2, cv=to_tf32):
    """the two post-network GEMMs: (r1 = relu(skip_r wp1^T + bp1), bound), and a function r1 -> (logits, bound)"""
    h1, bound = skip_gemm(skip_r, wp1, bp1, True, cv=cv)

    def logits(r1):
        return skip_gemm(r1, wp2, bp2, False, cv=cv)
    return (h1, bound), logits


# ------------------------------------------------------------------------------------------------------------------
# backward stages
# ------------------------------------------------------------------------------------------------------------------
def dz_all(dskip, wskip, cv=to_tf32):
    """dZ_all = dskip Wskip (B,T,L*R)"""
    acc, mag = _mm(dskip, wskip.t(), cv)
    return acc, lin_bound(mag, dskip.shape[-1])


def dz_block(dzall_l, dout, w2res, cv=to_tf32):
    """dz of one stack block = dZ_all[l] + dout W2res (dout None for the last block)"""
    dz = dzall_l.to(F64)
    if dout is None:
        return dz, torch.zeros_like(dz)
    acc, mag = _mm(dout, w2res.t(), cv)
    return dz + acc, lin_bound(mag, dout.shape[-1]) + U * (dz.abs() + acc.abs())


def dz_perblock(dout, dskip, w2, cv=to_tf32):
    """dz of the per-block backward = [dout | dskip] W2 (W2 = [W2res; W2skip], (R+S, R))"""
    R = w2.shape[1]
    acc, mag = _mm(dskip, w2[R:].t(), cv)
    K = dskip.shape[-1]
    if dout is not None:
        v, m = _mm(dout, w2[:R].t(), cv)
        acc, mag, K = acc + v, mag + m, K + R
    return acc, lin_bound(mag, K)


def gate_bwd(xin, haux, w1, b1, d, ks, dz, e_dz, cv=to_tf32, gate_fn=GATE_TANH_APPROX):
    """dpre (B,T,2R) = [d pre-sigmoid | d pre-tanh] from the recomputed gate and dz (known to within e_dz)"""
    pre, e = gate_pre(xin, haux, w1, b1, d, ks, cv)
    s, th, es, eth = _gate_parts(pre, e, gate_fn)
    dz = dz.to(F64)
    adz = dz.abs()
    ds = s * (1 - s)
    da = dz * th * ds
    dg = dz * s * (1 - th * th)
    eda = (th.abs() * ds * e_dz + adz * (ds * eth + th.abs() * (1 - 2 * s).abs() * es + th.abs() * es * es)
           + e_dz * (es + eth) + 6 * U * da.abs())
    edg = (s * (1 - th * th) * e_dz + adz * ((1 - th * th) * es + 2 * s * th.abs() * eth + s * eth * eth)
           + e_dz * (es + eth) + 6 * U * adz * s)
    return torch.cat([da, dg], -1), torch.cat([eda, edg], -1)


def dx_stage(dpre, w1, d, ks, dout=None, cv=to_tf32):
    """dxin = dout + sum_j dpre(t + (ks-1-j) d) W1[:, tap j]   (B,T,R)"""
    R = w1.shape[0] // 2
    acc, mag = 0, 0
    for j in range(ks):
        v, m = _mm(tshift(dpre, (ks - 1 - j) * d), w1[:, j * R:(j + 1) * R].t(), cv)
        acc, mag = acc + v, mag + m
    bound = lin_bound(mag, ks * 2 * R)
    if dout is None:
        return acc, bound + 0 * acc
    o = dout.to(F64)
    return acc + o, bound + U * (acc.abs() + o.abs())


def dhaux_stage(dpre, w1, ks, cv=to_tf32):
    """one block's contribution dpre(t) W1[:, aux] (B,T,Ap) and its bound (before the reduce-add)"""
    R = w1.shape[0] // 2
    acc, mag = _mm(dpre, w1[:, ks * R:].t(), cv)
    return acc, lin_bound(mag, 2 * R)


def accumulate(init, parts):
    """init + sum of (value, bound) parts, each added by one fp32 reduce-add; returns (ref, bound)"""
    out = init.to(F64).clone()
    bound = torch.zeros_like(out)
    for v, b in parts:
        out = out + v
        bound = bound + b + U * (out.abs() + v.abs())
    return out, bound


def wgrad(a, bs, init=None, db_init=None, cv=to_tf32, nsm=256):
    """C = init + sum_{b,t} A^T [B_0 | B_1 | ...] (M x N) and db = db_init + sum_{b,t} A (the all-ones column), with bounds.
    a (B,T,M); bs: list of (B,T,N_i) operands (already shifted).  The kernel sums B*T products per CTA range and then up
    to `nsm` slots in order, then adds into the caller's buffer."""
    A = cv(a).reshape(-1, a.shape[-1])
    Bm = torch.cat([cv(b).reshape(-1, b.shape[-1]) for b in bs], -1)
    K = A.shape[0] + nsm
    c = A.t() @ Bm
    cb = lin_bound(A.abs().t() @ Bm.abs(), K)
    db = A.sum(0)
    dbb = lin_bound(A.abs().sum(0), K)
    if init is not None:
        i = init.to(F64)
        c, cb = c + i, cb + U * ((c + i).abs() + i.abs())
    if db_init is not None:
        i = db_init.to(F64)
        db, dbb = db + i, dbb + U * ((db + i).abs() + i.abs())
    return (c, cb), (db, dbb)


def post_bwd(skip_r, r1, dlogits, dh1, wp1, wp2, cv=to_tf32):
    """post-network backward stages from the kernel's own inputs.  dh1 = (dlogits wp2) * (r1 > 0),
    dskip = (dh1 wp1) * (skip_r > 0) [dh1 = the kernel's, or None: the reference's], dWp2 = dlogits^T r1,
    dWp1 = dh1^T skip_r (+ bias sums).  Returns dict of name -> (ref, bound) (weight-gradient entries without init)."""
    out = {}
    acc, mag = _mm(dlogits, wp2.t(), cv)
    m = (r1 > 0).to(F64)
    out["dh1"] = (acc * m, lin_bound(mag, dlogits.shape[-1]) * m)
    if dh1 is None:
        dh1 = out["dh1"][0]
    acc, mag = _mm(dh1, wp1.t(), cv)
    m = (skip_r > 0).to(F64)
    out["dskip"] = (acc * m, lin_bound(mag, dh1.shape[-1]) * m)
    (out["dwp2"], out["dbp2"]) = wgrad(dlogits, [r1], cv=cv)
    (out["dwp1"], out["dbp1"]) = wgrad(dh1, [skip_r], cv=cv)
    return out


# ------------------------------------------------------------------------------------------------------------------
# reporting
# ------------------------------------------------------------------------------------------------------------------
def worst(got, ref, bound):
    """(largest err/bound, flat index of that element); NaN / inf in `got` count as infinitely wrong"""
    g = got.to(F64)
    err = (g - ref.to(F64)).abs()
    err = torch.where(torch.isfinite(g), err, torch.full_like(err, float("inf")))
    b = bound.to(F64)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / b.clamp_min(1e-300))
    i = int(torch.argmax(ratio.reshape(-1)))
    return float(ratio.reshape(-1)[i]), i


def locate(shape, i):
    """human-readable position of flat index i: (b, t, channel) with its 64-row tile and 32-column group for an
    activation, (row, column) with its 32-row / 32-column groups for a matrix"""
    idx = np.unravel_index(i, tuple(shape))
    if len(shape) == 3:
        b, t, c = (int(v) for v in idx)
        return "(b=%d, t=%d, ch=%d): time tile %d (rows %d..%d), column group %d" % (
            b, t, c, t // 64, t // 64 * 64, t // 64 * 64 + 63, c // 32)
    if len(shape) == 2:
        r, c = (int(v) for v in idx)
        return "(row=%d, col=%d): row group %d, column group %d" % (r, c, r // 32, c // 32)
    return "index %s" % (tuple(int(v) for v in idx),)


def assert_within(got, ref, bound, what):
    """assert |got - ref| <= bound element-wise; returns the largest err/bound.  The failure message names the worst
    element, its 64-row time tile and its 32-column group."""
    assert tuple(got.shape) == tuple(ref.shape), (what, tuple(got.shape), tuple(ref.shape))
    r, i = worst(got, ref, bound)
    if not r <= 1.0:
        g = float(got.reshape(-1)[i])
        rf = float(ref.reshape(-1)[i])
        bd = float(bound.reshape(-1)[i])
        raise AssertionError("%s: err/bound %.3g at %s; got %.9g, ref %.9g, bound %.3g" % (
            what, r, locate(got.shape, i), g, rf, bd))
    return r
