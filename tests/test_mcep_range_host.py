# -*- coding: utf-8 -*-
"""CPU tier: the claim that bounds wnb_mcep's supported range (include/wnb200.h: fftl a power of two from 1024 to 4096,
order <= 40, 0 <= alpha <= 0.6, "there the bin sums equal SPTK's truncated recursions to 1e-13"), which the GPU bar of
tests/mcep_check.py rests on.  The kernel evaluates every frequency warp as a sum over the fftl / 2 + 1 bins; the oracle
runs SPTK's FFTs and the freqt / frqtr recursions, which truncate at fftl / 2 terms.  Both are compared here with the
direct sums on the warped axis, evaluated in extended precision by the Chebyshev recurrence from the kernel's own
cos w~ table (utils.mcep.warped_cos), at every corner of the range:
  * warped autocorrelations: MO.frqtr(rho[0 .. L/2], 2 order, alpha), rho = Re IDFT(R) as the oracle forms it, against
    r(j) = (1/L) sum_k mult_k R_k T_j(cos w~_k), to 1e-13 relative to r(0), on Hamming-windowed speech-like and
    full-scale square-wave frames (R their periodograms);
  * log|H|: Re DFT of MO.freqt(c, L/2, -alpha) zero-padded to L against sum_m c_m T_m(cos w~_k), to 1e-13 absolute,
    for random decaying c.
Below the range the recursions' truncation shows: at fftl 512, alpha 0.6, order 40 frqtr is off by more than 1e-6, and
the library rejects fftl 512."""
import numpy as np

from oracle import mcep_oracle as MO
from tests.mcep_check import _speechlike

LD = np.longdouble
FFTLS = (1024, 2048, 4096)
ALPHAS = (0.0, 0.41, 0.455, 0.6)
ORDERS = (1, 24, 35, 40)
BAR = 1e-13


def _frames(L):
    """three Hamming-windowed speech-like frames and two full-scale square waves (periods 37 and 100 samples)"""
    rng = np.random.RandomState(L)
    w = MO.hamming(L)
    x = _speechlike(rng, 4 * L)
    n = np.arange(L)
    return [x[t * L // 2:t * L // 2 + L] * w for t in range(3)] + \
        [np.where((n // p) % 2 == 0, 32767.0, -32768.0) * w for p in (37, 100)]


def _chebyshev(cw, n):
    """T_0 .. T_n at every bin, in extended precision, by T_{j+1} = 2 x T_j - T_{j-1}: (n + 1, bins)"""
    x = np.asarray(cw, dtype=LD)
    T = np.empty((n + 1, len(x)), dtype=LD)
    T[0] = 1
    if n >= 1:
        T[1] = x
    for j in range(1, n):
        T[j + 1] = 2 * x * T[j] - T[j - 1]
    return T


def _frqtr_error(L, alpha, order, frame):
    """max_j |frqtr(rho)_j - (1/L) sum_k mult_k R_k T_j(cos w~_k)| / r(0) for the frame's periodogram R"""
    from pytorchwavenetvocoder_b200.utils.mcep import warped_cos
    nb = L // 2 + 1
    R = np.abs(np.fft.fft(frame)) ** 2 + MO.EPS
    rho = np.real(np.fft.ifft(R))[:nb]
    got = MO.frqtr(rho, 2 * order, alpha)
    mult = np.full(nb, 2, dtype=LD)
    mult[0] = mult[-1] = 1
    want = _chebyshev(warped_cos(L, alpha), 2 * order) @ (mult * R[:nb].astype(LD)) / LD(L)
    return float(np.max(np.abs(got.astype(LD) - want)) / want[0])


def _log_h_error(L, alpha, order, c):
    """max_k |Re DFT(freqt(c, L/2, -alpha), zero-padded to L)_k - sum_m c_m T_m(cos w~_k)| over k = 0 .. L/2"""
    from pytorchwavenetvocoder_b200.utils.mcep import warped_cos
    nb = L // 2 + 1
    g = np.zeros(L)
    g[:nb] = MO.freqt(c, L // 2, -alpha)
    got = np.real(np.fft.fft(g))[:nb]
    want = np.asarray(c, dtype=LD) @ _chebyshev(warped_cos(L, alpha), order)
    return float(np.max(np.abs(got.astype(LD) - want)))


def test_bin_sums_equal_the_recursions_inside_the_range():
    worst_r = worst_h = (-1.0, "")
    bad = []
    for fftl in FFTLS:
        frames = _frames(fftl)
        for alpha in ALPHAS:
            for order in ORDERS:
                rng = np.random.RandomState(fftl + order)
                er = max(_frqtr_error(fftl, alpha, order, f) for f in frames)
                eh = 0.0
                for _ in range(3):
                    c = rng.randn(order + 1) * 0.6 / np.arange(1, order + 2)
                    c[0] = 4.0
                    eh = max(eh, _log_h_error(fftl, alpha, order, c))
                where = "fftl %d alpha %g order %d" % (fftl, alpha, order)
                worst_r, worst_h = max(worst_r, (er, where)), max(worst_h, (eh, where))
                if er > BAR or eh > BAR:
                    bad.append("%s: frqtr %.2e of r(0), log|H| %.2e" % (where, er, eh))
    print("inside the range: worst frqtr %.2e of r(0) (%s), worst log|H| %.2e (%s)" % (worst_r + worst_h))
    assert not bad, bad


def test_fftl_512_is_outside_the_range():
    """At fftl 512 the truncated frqtr departs from the bin sums (here by far more than the GPU bar could absorb), so
    the library must keep rejecting it."""
    from pytorchwavenetvocoder_b200._lib import load
    from tests.test_mcep_host import WNB_ERR_UNSUPPORTED, _call
    err = max(_frqtr_error(512, 0.6, 40, f) for f in _frames(512))
    print("fftl 512 alpha 0.6 order 40: frqtr %.2e of r(0)" % err)
    assert err > 1e-6
    lib = load()
    assert _call(lib, fftl=512, order=40, alpha=0.6) == WNB_ERR_UNSUPPORTED
    assert b"not supported" in lib.wnb_last_error()
