# -*- coding: utf-8 -*-
"""float64 restatement of one ``wnb_adam_flat`` step (csrc/adam.cu) with a first-order error bound per element, used by
tests/test_gpu_optim.py and checked on the CPU by tests/test_train_batch_adam_reference.py.

The launcher rounds its scalars to float32 once (from double, as torch does); the reference takes those same float32
scalars and the kernel's fp32 inputs and evaluates the step exactly (to float64):

    g' = g + wd*p                      (only when wd != 0)
    m' = m + omb1*(g' - m)
    v' = b2*v + omb2*g'*g'
    p' = p - step * m' / (sqrt(v') / bc2s + eps)

Every fp32 add, multiply, divide, sqrtf or fma of the kernel is correctly rounded (nvcc --fmad=true, no fast-math), so
each one adds at most u = 2^-24 of its result -- or, for a result in the subnormal range, half the smallest subnormal
(eta = 2^-150).  The bound below covers both the separately rounded and the fma-contracted form of every operation and
propagates the input errors to first order.
"""
import math

import numpy as np

U32 = 2.0 ** -24
ETA = 2.0 ** -150


def scalars(lr, betas, eps, wd, bc1, bc2):
    """the float32 scalars wnb_adam_flat hands its kernel"""
    b1, b2 = betas
    f = lambda z: float(np.float32(z))  # noqa: E731
    return dict(step=f(lr / bc1), omb1=f(1.0 - b1), b2=f(b2), omb2=f(1.0 - b2), eps=f(eps), wd=f(wd),
                bc2s=f(math.sqrt(bc2)))


def bias_corrections(betas, k):
    """(1 - b1^k, 1 - b2^k) as optim.Adam computes them in Python floats"""
    return 1.0 - betas[0] ** k, 1.0 - betas[1] ** k


def adam_step(p, g, m, v, sc, eps_first=False):
    """float64 values and bounds of one step: dict(p=, m=, v=) and dict of the same keys with the error bounds.
    eps_first=True restates a wrong order of operations ((sqrt(v') + eps) / bc2s) for the checks of the checker."""
    p, g, m, v = (np.asarray(a, dtype=np.float64) for a in (p, g, m, v))
    u, eta = U32, ETA
    step, omb1, b2, omb2, eps, wd, bc2s = (sc[k] for k in ("step", "omb1", "b2", "omb2", "eps", "wd", "bc2s"))
    if wd != 0.0:
        wp = wd * p
        gg = g + wp
        e_g = 2 * u * (np.abs(wp) + np.abs(gg)) + 2 * eta
    else:
        gg, e_g = g, np.zeros_like(g)
    dm = omb1 * (gg - m)
    m1 = m + dm
    e_m = abs(omb1) * e_g + u * (2 * np.abs(dm) + np.abs(m1)) + 3 * eta
    og = omb2 * gg
    og2 = og * gg
    bv = b2 * v
    v1 = bv + og2
    e_v = 2 * np.abs(og) * e_g + u * (2 * np.abs(og2) + np.abs(bv) + np.abs(v1)) + 4 * eta
    r = np.sqrt(v1)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_r = np.minimum(np.where(r > 0, e_v / (2 * r), np.inf), np.sqrt(e_v))
    if eps_first:
        den = (r + eps) / bc2s
        e_den = e_r / bc2s + 2 * u * den + 2 * eta
    else:
        s = r / bc2s
        e_s = e_r / bc2s + 2 * u * s + 2 * eta
        den = s + eps
        e_den = e_s + u * den + eta
    q = m1 / den
    e_q = (e_m + np.abs(q) * e_den) / (den - e_den) + u * np.abs(q) + eta
    sq = step * q
    p1 = p - sq
    e_p = step * e_q + u * (np.abs(sq) + np.abs(p1)) + 2 * eta
    return dict(p=p1, m=m1, v=v1), dict(p=e_p, m=e_m, v=e_v)


def emulate_fp32(p, g, m, v, sc, eps_first=False, contract=False):
    """the kernel's arithmetic in numpy float32 (contract=True: the fma-contracted form, each fma evaluated exactly in
    float64 and rounded once -- exact for products of two floats), for the checks of the bound on the CPU"""
    f32 = np.float32
    p, g, m, v = (np.asarray(a, dtype=f32) for a in (p, g, m, v))
    step, omb1, b2, omb2, eps, wd, bc2s = (f32(sc[k]) for k in ("step", "omb1", "b2", "omb2", "eps", "wd", "bc2s"))

    def fma(a, b, c):
        return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)

    if wd != 0:
        g = fma(p, wd, g) if contract else g + wd * p
    m1 = fma(g - m, omb1, m) if contract else m + omb1 * (g - m)
    og = omb2 * g
    v1 = fma(v, b2, og * g) if contract else b2 * v + og * g
    s = np.sqrt(v1)
    den = (s + eps) / bc2s if eps_first else s / bc2s + eps
    q = m1 / den
    p1 = fma(q, -step, p) if contract else p - step * q
    return dict(p=p1, m=m1, v=v1)


def ratios(got, ref, bound):
    """largest err/bound of each output (an exact result where the bound is 0 counts as 0) and the index of the worst"""
    out = {}
    for k in ("p", "m", "v"):
        err = np.abs(np.asarray(got[k], dtype=np.float64) - ref[k])
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err == 0, 0.0, err / bound[k])
        r = np.where(np.isnan(r), np.inf, r)
        i = int(np.argmax(r))
        out[k] = (float(r[i]), i)
    return out


def spread_inputs(n, seed, wd_zero_p=True):
    """fp32 p, g, m, v over many magnitudes and both signs: |g| from 1e-20 to 1e3; every 5th element a first step
    (m = v = 0, g != 0); every 7th g = m = v = 0; every 11th p = 0"""
    rng = np.random.RandomState(seed)
    sgn = lambda: np.where(rng.rand(n) < 0.5, -1.0, 1.0)  # noqa: E731
    g = sgn() * 10.0 ** rng.uniform(-20, 3, n)
    m = sgn() * 10.0 ** rng.uniform(-20, 3, n) * (rng.rand(n) < 0.8)
    v = 10.0 ** rng.uniform(-40, 6, n) * (rng.rand(n) < 0.9)
    m = np.where(rng.rand(n) < 0.3, g * rng.uniform(-2, 2, n), m)     # moments of the gradient's own size
    v = np.where(rng.rand(n) < 0.3, g * g * rng.uniform(0, 3, n), v)
    p = sgn() * 10.0 ** rng.uniform(-8, 2, n)
    i = np.arange(n)
    m[i % 5 == 1], v[i % 5 == 1] = 0.0, 0.0
    g[i % 7 == 2], m[i % 7 == 2], v[i % 7 == 2] = 0.0, 0.0, 0.0
    if wd_zero_p:
        p[i % 11 == 3] = 0.0
    return tuple(a.astype(np.float32) for a in (p, g, m, v))
