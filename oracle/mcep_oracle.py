# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE (oracle): ctypes front end of oracle/mcep_oracle.c, the CPU restatement of the reference's
pysptk-based mel-cepstral analysis (reference bin/feature_extract.py:33-52 ``stft_mcep``).  See the header of the C
file: parity is UNPINNED against pysptk (absent from this image); the restatement is pinned by exact-model recovery,
the criterion's stationarity condition and the other properties checked in tests/test_mcep_oracle.py.

Only tests/, __graft_entry__.smoke() and tools/ may import this module."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "mcep_oracle.c")
LIB = os.path.join(HERE, "_build", "libmcep_oracle.so")
_lib = None

EPS = 1e-10          # the reference's pysptk.mcep(..., eps=1e-10, etype=1)
MINITER, MAXITER, THRESHOLD, MIN_DET = 2, 30, 1e-3, 1e-6      # pysptk's defaults


def build(force=False):
    """gcc -O2 -ffp-contract=off -> oracle/_build/"""
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", LIB, SRC, "-lm"])
    return LIB


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        d, i, f = ctypes.POINTER(ctypes.c_double), ctypes.c_int, ctypes.c_double
        L.mcep_freqt.argtypes = [d, i, d, i, f]
        L.mcep_frqtr.argtypes = [d, i, d, i, f]
        L.mcep_frame.argtypes = [d, i, i, f, i, i, f, f, f, i, d, d]
        L.mcep_frame.restype = i
        L.mcep_initial.argtypes = [d, i, i, f, f, d, d]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def freqt(c, order, alpha):
    """SPTK freqt: c[0..m1] -> order + 1 coefficients on the axis warped by alpha."""
    c = np.ascontiguousarray(c, dtype=np.float64)
    out = np.empty(order + 1, dtype=np.float64)
    lib().mcep_freqt(_p(c), len(c) - 1, _p(out), int(order), float(alpha))
    return out


def frqtr(rho, order, alpha):
    """SPTK frqtr: rho[0..L/2] -> r(0..order), r(j) = (1/L) sum_k R_k cos(j w~_k)."""
    rho = np.ascontiguousarray(rho, dtype=np.float64)
    out = np.empty(order + 1, dtype=np.float64)
    lib().mcep_frqtr(_p(rho), len(rho) - 1, _p(out), int(order), float(alpha))
    return out


def mcep(frame, order, alpha, eps=EPS, miniter=MINITER, maxiter=MAXITER, threshold=THRESHOLD, min_det=MIN_DET,
         force_iters=None):
    """pysptk.mcep(frame, order, alpha, eps=eps, etype=1) of one windowed frame (length a power of two).

    Returns (mc float64 (order + 1,), count, stats): count is the number of Newton updates applied (negative -j: the
    solve of iteration j failed); stats[j] is the convergence statistic of iteration j (NaN where none was computed).
    force_iters runs exactly that many updates with no convergence exit."""
    x = np.ascontiguousarray(frame, dtype=np.float64)
    L = len(x)
    assert L >= 2 and L & (L - 1) == 0, "frame length must be a power of two"
    force = -1 if force_iters is None else int(force_iters)
    mc = np.empty(order + 1, dtype=np.float64)
    stats = np.empty(max(maxiter, force) + 1, dtype=np.float64)
    n = lib().mcep_frame(_p(x), L, int(order), float(alpha), int(miniter), int(maxiter), float(threshold), float(eps),
                         float(min_det), force, _p(mc), _p(stats))
    return mc, int(n), stats


def initial_value(frame, order, alpha, eps=EPS):
    """The Newton start alone: freqt of the halved real cepstrum of log(|X|^2 + eps), and the convergence seed s."""
    x = np.ascontiguousarray(frame, dtype=np.float64)
    mc = np.empty(order + 1, dtype=np.float64)
    s = np.zeros(1, dtype=np.float64)
    lib().mcep_initial(_p(x), len(x), int(order), float(alpha), float(eps), _p(mc), _p(s))
    return mc, float(s[0])


def hamming(fftl):
    """``scipy.signal.get_window("hamming", fftl)``: the periodic Hamming window."""
    from scipy.signal import get_window
    return np.ascontiguousarray(get_window("hamming", fftl), dtype=np.float64)


def n_frames(n_samples, fftl, hop):
    """Frames of stft_mcep: ``(len - fftl) // hop + 1`` (no padding), 0 when the signal is shorter than fftl."""
    return max(0, (int(n_samples) - int(fftl)) // int(hop) + 1)


def frames(x, fftl, hop):
    """stft_mcep's framing: frame i is x[hop i : hop i + fftl] in int16 units, times the periodic Hamming window."""
    x = np.asarray(x, dtype=np.float64)
    n = n_frames(len(x), fftl, hop)
    idx = np.arange(n)[:, None] * hop + np.arange(fftl)[None, :]
    return x[idx] * hamming(fftl)[None, :]


def stft_mcep(x, fftl, hop, order, alpha, **kw):
    """reference feature_extract.py:33-52 on one signal (int16 or float64 samples): (frames, order + 1) float64, the
    per-frame counts and statistics.  kw goes to ``mcep`` (force_iters may be a per-frame sequence)."""
    fr = frames(x, fftl, hop)
    force = kw.pop("force_iters", None)
    out, counts, stats = [], [], []
    for i, f in enumerate(fr):
        fi = force[i] if force is not None and np.ndim(force) else force
        mc, n, st = mcep(f, order, alpha, force_iters=fi, **kw)
        out.append(mc)
        counts.append(n)
        stats.append(st)
    return np.array(out).reshape(len(fr), order + 1), np.array(counts, dtype=np.int64), stats
