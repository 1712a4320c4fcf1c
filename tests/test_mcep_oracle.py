# -*- coding: utf-8 -*-
"""CPU tier: oracle/mcep_oracle.c, the restatement of SPTK's mcep that the GPU mel-cepstra are checked against, pinned
by what mel-cepstral analysis is.  Every property below is evaluated with direct numpy cosines on the alpha-warped axis,
independent of the oracle's freqt, frqtr and Cholesky solve."""
import numpy as np
import pytest
from scipy.signal import get_window, lfilter

from oracle import mcep_oracle as MO

EPS = 1e-10


def _warped(L, a):
    """w~_k for all L bins: the phase of the all-pass (z^-1 - a) / (1 - a z^-1) at w_k = 2 pi k / L."""
    w = 2 * np.pi * np.arange(L) / L
    return np.arctan2((1 - a * a) * np.sin(w), (1 + a * a) * np.cos(w) - 2 * a)


def _log_h2(c, th):
    return 2.0 * np.cos(np.outer(th, np.arange(len(c)))) @ c


def _model_frame(cstar, L, a):
    """the zero-phase frame whose periodogram plus eps is exp(2 sum c*_m cos(m w~_k))"""
    P = np.exp(_log_h2(cstar, _warped(L, a))) - EPS
    return np.fft.irfft(np.sqrt(P[:L // 2 + 1]), L)


def _cstar(M, seed, c0=4.0):
    rng = np.random.RandomState(seed)
    c = rng.randn(M + 1) * 0.6 / np.arange(1, M + 2)
    c[0] = c0
    return c


def _speechlike(seed, n):
    rng = np.random.RandomState(seed)
    e = rng.randn(n) * 400.0
    e[::97] += 6000.0                             # a 165 Hz pulse train at 16 kHz
    return lfilter([1.0], [1.0, -1.3, 0.8, -0.2], e)


@pytest.mark.parametrize("M,a,L", [(12, 0.0, 512), (24, 0.41, 1024), (25, 0.41, 1024), (35, 0.455, 1024),
                                   (25, 0.55, 2048), (12, 0.55, 512), (35, 0.0, 2048), (24, 0.455, 2048)])
def test_exact_model_recovery(M, a, L):
    cs = _cstar(M, M + L)
    x = _model_frame(cs, L, a)
    mc, n, _ = MO.mcep(x, M, a, threshold=1e-14, maxiter=100)
    assert n >= 0
    assert np.abs(mc - cs).max() < 1e-8, np.abs(mc - cs).max()
    if a == 0.0:
        mi, _ = MO.initial_value(x, M, a)
        assert np.abs(mi - cs).max() < 1e-12      # the cepstrum halving and freqt's conventions


def test_warped_cosine_mean_identity():
    th = _warped(1024, 0.41)
    for m in range(80):
        assert abs(np.mean(np.cos(m * th)) - (-0.41) ** m) < 1e-15


@pytest.mark.parametrize("M,a,L,seed", [(24, 0.41, 1024, 0), (25, 0.41, 1024, 1), (35, 0.455, 1024, 2),
                                        (25, 0.55, 2048, 3)])
def test_stationarity_and_minimum(M, a, L, seed):
    """At the returned c: (1/L) sum_k cos(m w~_k) P_k / |H_k|^2 = (-a)^m for m = 0..M, and E(c +- h e_m) > E(c)."""
    x = _speechlike(seed, 4 * L)
    th = _warped(L, a)
    P = np.abs(np.fft.fft(MO.frames(x, L, L)[2])) ** 2 + EPS
    mc, n, _ = MO.mcep(MO.frames(x, L, L)[2], M, a, threshold=1e-13, maxiter=200)
    assert n >= 0
    cosm = np.cos(np.outer(th, np.arange(M + 1)))
    R = P / np.exp(2.0 * cosm @ mc)
    lhs = (cosm * R[:, None]).mean(axis=0)
    assert np.abs(lhs - (-a) ** np.arange(M + 1)).max() < 1e-10

    def E(c):
        q = P / np.exp(2.0 * cosm @ c)
        return np.sum(q - np.log(q) - 1.0)
    e0 = E(mc)
    for m in range(M + 1):
        for h in (1e-4, -1e-4):
            c = mc.copy()
            c[m] += h
            assert E(c) > e0, (m, h)


def test_digital_silence():
    for M, a in ((24, 0.41), (35, 0.455)):
        mc, n, _ = MO.mcep(np.zeros(1024), M, a)
        assert n >= 0
        assert abs(mc[0] - 0.5 * np.log(EPS)) < 1e-12 and np.abs(mc[1:]).max() < 1e-12


def test_gain_adds_k_log2_to_c0_only():
    x = MO.frames(_speechlike(5, 4096), 1024, 1024)[1]
    base, n0, _ = MO.mcep(x, 25, 0.41, threshold=1e-12, maxiter=100)
    for k in (-3, 1, 4):
        mc, n, _ = MO.mcep(x * 2.0 ** k, 25, 0.41, threshold=1e-12, maxiter=100)
        d = mc - base
        assert abs(d[0] - k * np.log(2.0)) < 1e-9 and np.abs(d[1:]).max() < 1e-9, (k, d[:3])


@pytest.mark.parametrize("fftl,hop", [(1024, 80), (1024, 256), (512, 80)])
def test_framing(fftl, hop):
    w = get_window("hamming", fftl)
    assert np.abs(w - (0.54 - 0.46 * np.cos(2 * np.pi * np.arange(fftl) / fftl))).max() < 1e-15   # periodic
    for n in (fftl - 1, fftl, fftl + 1, fftl + hop - 1, fftl + hop, fftl + 5 * hop + 3):
        want = (n - fftl) // hop + 1 if n >= fftl else 0
        assert MO.n_frames(n, fftl, hop) == want
        x = np.arange(n, dtype=np.float64)
        fr = MO.frames(x, fftl, hop)
        assert fr.shape == (want, fftl)
        for i in range(len(fr)):
            assert np.array_equal(fr[i], x[hop * i:hop * i + fftl] * w)


def test_counts_statistics_and_forcing():
    """The count is the number of updates; stats[j] records |(r0_j - s) / r0_j| from miniter on; the converged frame
    equals the same frame forced to that count; maxiter caps the updates."""
    x = MO.frames(_speechlike(7, 4096), 1024, 80)[3]
    mc, n, st = MO.mcep(x, 25, 0.41)
    assert 1 <= n < 30 and st[n + 1] < 1e-3 and np.all(st[2:n + 1] >= 1e-3) and np.isnan(st[:2]).all()
    forced, nf, _ = MO.mcep(x, 25, 0.41, force_iters=n)
    assert nf == n and np.array_equal(forced, mc)
    capped, nc, _ = MO.mcep(x, 25, 0.41, maxiter=1)
    assert nc == 1 and np.array_equal(capped, MO.mcep(x, 25, 0.41, force_iters=1)[0])


def test_against_pysptk_when_importable():
    pysptk = pytest.importorskip("pysptk")
    x = _speechlike(9, 16000)
    fr = MO.frames(x, 1024, 80)[:40]
    for f in fr:
        want = pysptk.mcep(f, 25, 0.41, eps=1e-10, etype=1)
        got, _, _ = MO.mcep(f, 25, 0.41)
        assert np.abs(got - want).max() < 1e-6 * (1 + np.abs(want).max())
