# -*- coding: utf-8 -*-
"""GPU tier: wnb_mcep at the corners of its supported range and at every exit of its Newton loop, frame by frame
against oracle/mcep_oracle.c with the checker and bar of tests/mcep_check.py.

  * range corners: fftl 4096 (the largest shared-memory footprint; thread 0 takes 9 bins, the half-weight bin
    fftl / 2 among them), fftl 1024 at alpha 0.6 and order 40, alpha 0 at order 40, orders 1, 3 and 4 (2 order + 1
    values of r on either side of the kernel's chunk of 8) and 31, 32 and 33 (order + 1 on either side of the 32 lanes of
    the one-warp Cholesky factorisation);
  * loop exits through mcep_batch: maxiter 0 (the initial value as is), maxiter 1, threshold 0 (never converges, up to
    WNB_MCEP_MAX_ITER updates), miniter 0 and 1 (the convergence seed, row order + 1 of the initial-value map, compared
    at the first iteration), miniter above maxiter, a threshold every frame meets at the first test;
  * failed solves through wnb_mcep called directly (mcep_batch fixes min_det): at the first iteration, at every later
    iteration a frame's pivots can fail at, and the host's error naming the utterance and the frame;
  * the frame-to-utterance search over 1, 2, 3 and 257 utterances: each utterance's rows and counts bit-identical to
    running it alone."""
import numpy as np
import pytest

from oracle import mcep_oracle as MO
from tests.mcep_check import _allowed, _check, _speechlike, mcep_direct

pytestmark = pytest.mark.gpu
FS = 16000


def _ragged(rng, fftl, hop, as_int16, long_len=20000):
    """speech-like utterances of lengths fftl, fftl + 1, fftl + hop - 1, fftl + hop and long_len, as int16 or as float64
    in int16 units with a sub-LSB offset"""
    xs = [_speechlike(rng, n) for n in (fftl, fftl + 1, fftl + hop - 1, fftl + hop, long_len)]
    if as_int16:
        return [np.int16(x) for x in xs]
    return [np.float64(np.int16(x)) + rng.uniform(-0.5, 0.5, len(x)) for x in xs]


def _check_ragged(xs, fftl, hop, order, alpha, cutoff, label, **loop):
    """every frame of the four short utterances and about 20 frames of the long one"""
    _check(xs, FS, fftl, hop, order, alpha, cutoff, which=range(4), label=label + " short", **loop)
    stride = max(1, MO.n_frames(len(xs[4]), fftl, hop) // 20)
    _check(xs, FS, fftl, hop, order, alpha, cutoff, which=[4], stride=stride,
           label="%s long (every %d-th frame)" % (label, stride), **loop)


CORNERS = [(4096, 80, 40, 0.6), (4096, 256, 40, 0.6), (4096, 80, 24, 0.41), (4096, 256, 24, 0.41),
           (1024, 80, 40, 0.6), (1024, 80, 40, 0.0), (4096, 80, 40, 0.0)] + \
          [(1024, 80, m, 0.41) for m in (1, 3, 4, 31, 32, 33)]


@pytest.mark.parametrize("fftl,hop,order,alpha", CORNERS)
@pytest.mark.parametrize("as_int16", [True, False])
def test_range_corners(fftl, hop, order, alpha, as_int16):
    """int16 input without a cutoff, float64 input through the low-cut filter at 70 Hz"""
    rng = np.random.RandomState(fftl + 7 * hop + 11 * order + int(100 * alpha) + as_int16)
    xs = _ragged(rng, fftl, hop, as_int16)
    cutoff = 0 if as_int16 else 70
    _check_ragged(xs, fftl, hop, order, alpha, cutoff, "fftl %d hop %d order %d alpha %g cutoff %d %s"
                  % (fftl, hop, order, alpha, cutoff, "int16" if as_int16 else "float64"))


def test_fftl_512_is_rejected():
    """the recursions the bar rests on break down below fftl 1024 (tests/test_mcep_range_host.py)"""
    from pytorchwavenetvocoder_b200._lib import WnbError
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    with pytest.raises(WnbError, match="not supported"):
        mcep_batch([np.zeros(2000, np.int16)], FS, 512, 80, 40, 0.6)


# ---------------------------------------------------------------------------------------------- exits of the loop
def _arctic_batch(seed, as_int16=True):
    rng = np.random.RandomState(seed)
    return _ragged(rng, 1024, 80, as_int16, long_len=4000)


def test_maxiter_0_returns_the_initial_value():
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    xs = _arctic_batch(40)
    hist = _check(xs, FS, 1024, 80, 25, 0.41, maxiter=0, label="maxiter 0")
    assert set(hist) == {0}, hist
    feats = mcep_batch(xs, FS, 1024, 80, 25, 0.41, maxiter=0)
    for u, x in enumerate(xs):
        for t, fr in enumerate(MO.frames(x, 1024, 80)):
            ok, _ = _allowed(feats[u][t], MO.initial_value(fr, 25, 0.41)[0])
            assert ok.all(), (u, t, feats[u][t], MO.initial_value(fr, 25, 0.41)[0])


def test_maxiter_1():
    hist = _check(_arctic_batch(41), FS, 1024, 80, 25, 0.41, maxiter=1, label="maxiter 1")
    assert set(hist) == {1}, hist


def test_threshold_0_never_converges():
    xs = _arctic_batch(42, as_int16=False)
    hist = _check(xs, FS, 1024, 80, 25, 0.41, 70, threshold=0.0, label="threshold 0 maxiter 30")
    assert set(hist) == {30}, hist
    rng = np.random.RandomState(43)
    xs = [np.int16(_speechlike(rng, 1024)) for _ in range(3)]
    hist = _check(xs, FS, 1024, 80, 25, 0.41, threshold=0.0, maxiter=1000, label="threshold 0 maxiter 1000")
    assert set(hist) == {1000}, hist


def _seed_tuned_frames(rng, order, alpha, rel):
    """one-frame float64 utterances scaled so that the convergence seed s (the halved cepstrum's c[0]; it moves by
    log g under a gain g) lies at r0 (1 + rel) for each rel, r0 the zeroth warped autocorrelation of the first iteration
    (gain invariant), evaluated with direct cosines.  The first test then gives |(r0 - s) / r0| ~ |rel|.  Also returns
    |mc[0] - s|: how far row 0 of the initial-value map lies from the seed row."""
    L = 1024
    w = 2 * np.pi * np.arange(L) / L
    th = np.arctan2((1 - alpha * alpha) * np.sin(w), (1 + alpha * alpha) * np.cos(w) - 2 * alpha)
    cosm = np.cos(np.outer(th, np.arange(order + 1)))
    x = _speechlike(rng, L + 80 * len(rel))
    xs, gap = [], []
    for i, d in enumerate(rel):
        seg = x[80 * i:80 * i + L]
        mc, s = MO.initial_value(seg * MO.hamming(L), order, alpha)
        P = np.abs(np.fft.fft(seg * MO.hamming(L))) ** 2 + MO.EPS
        r0 = np.mean(P / np.exp(2.0 * cosm @ mc))
        xs.append(seg * np.exp(r0 * (1 + d) - s))
        gap.append(abs(mc[0] - s))
    return xs, gap


@pytest.mark.parametrize("miniter", [0, 1])
def test_seed_is_compared_at_the_first_iteration(miniter):
    """miniter 0 and 1 test convergence at j = 1 against the seed; at alpha 0.41 the seed row differs from row 0, so a
    frame whose seed sits within the threshold of r0 stops with no update only if the kernel read the right row"""
    rel = [1e-5, 3e-4, -3e-4, 3e-3, -3e-3, 0.3]
    xs, gap = _seed_tuned_frames(np.random.RandomState(44), 25, 0.41, rel)
    assert min(gap) > 100 * 1e-3, gap
    hist = _check(xs, FS, 1024, 80, 25, 0.41, miniter=miniter, label="miniter %d, seed within 1e-5 ... 0.3 of r0"
                  % miniter)
    assert hist.get(0) == 3 and sum(hist.values()) == len(rel), hist


@pytest.mark.parametrize("miniter,maxiter", [(5, 3), (31, 30)])
def test_miniter_above_maxiter(miniter, maxiter):
    hist = _check(_arctic_batch(45), FS, 1024, 80, 25, 0.41, miniter=miniter, maxiter=maxiter,
                  label="miniter %d maxiter %d" % (miniter, maxiter))
    assert set(hist) == {maxiter}, hist


@pytest.mark.parametrize("miniter", [1, 2, 5])
def test_every_frame_stops_at_miniter(miniter):
    hist = _check(_arctic_batch(46 + miniter), FS, 1024, 80, 25, 0.41, miniter=miniter, threshold=1e30,
                  label="threshold 1e30 miniter %d" % miniter)
    assert set(hist) == {miniter - 1}, hist


# -------------------------------------------------------------------------------------------------- failed solves
def test_solve_fails_at_the_first_iteration():
    xs = _arctic_batch(50)
    hist = _check(xs, FS, 1024, 80, 25, 0.41, min_det=1e300, label="min_det 1e300")
    assert set(hist) == {-1}, hist
    feats, _ = mcep_direct(xs, 1024, 80, 25, 0.41, min_det=1e300)
    for u, x in enumerate(xs):
        for t, fr in enumerate(MO.frames(x, 1024, 80)):
            assert _allowed(feats[u][t], MO.initial_value(fr, 25, 0.41)[0])[0].all(), (u, t)


def _first_failure(frame, order, alpha, lo, hi=1e300):
    """bisect min_det on the oracle between lo and hi, whose counts differ: the switch point (the lowest min_det found
    whose count differs from lo's), to 64 halvings of log(hi / lo)"""
    c_lo = MO.mcep(frame, order, alpha, min_det=lo)[1]
    assert MO.mcep(frame, order, alpha, min_det=hi)[1] != c_lo
    for _ in range(64):
        mid = np.exp(0.5 * (np.log(lo) + np.log(hi)))
        if MO.mcep(frame, order, alpha, min_det=mid)[1] == c_lo:
            lo = mid
        else:
            hi = mid
    return hi


def _switch_points(frame, order, alpha):
    """every min_det where the oracle's count changes, from pysptk's 1e-6 (a normal solve) up to count -1: the pivots
    of the iterations, in increasing order"""
    pts, lo = [], 1e-6
    while MO.mcep(frame, order, alpha, min_det=lo)[1] != -1:
        b = _first_failure(frame, order, alpha, lo)
        pts.append(b)
        lo = b * (1 + 1e-6)
        assert len(pts) < 40
    return pts


def test_solve_fails_at_later_iterations():
    """For two frames, min_det at 1 -+ 1e-6 of every switch point of the oracle's count (far from the ~1e-12 by which
    the kernel's pivots differ from the oracle's): on each side the kernel takes the oracle's count, from a normal solve
    through -j for j from the frame's last update down to 1, and the row after j - 1 updates"""
    rng = np.random.RandomState(51)
    x = _speechlike(rng, 1024 + 80 * 7)
    seen = set()
    for t in (2, 7):
        seg = [np.int16(x[80 * t:80 * t + 1024])]
        fr = MO.frames(seg[0], 1024, 80)[0]
        pts = _switch_points(fr, 25, 0.41)
        for b in pts:
            below, above = b * (1 - 1e-6), b * (1 + 1e-6)
            for md in (below, above):
                h = _check(seg, FS, 1024, 80, 25, 0.41, min_det=md, label="frame %d min_det %.17g" % (t, md))
                seen.update(h)
            mc_above, n_above, _ = MO.mcep(fr, 25, 0.41, min_det=above)
            assert n_above < 0 and np.array_equal(mc_above, MO.mcep(fr, 25, 0.41, force_iters=-n_above - 1)[0])
    assert -1 in seen and min(seen) <= -2 and max(seen) > 0, seen


def test_failed_solve_error_names_utterance_and_frame(monkeypatch):
    """A failed solve in a frame past the first of an utterance past the first: mcep_batch names that frame, its
    utterance and the iteration.  min_det sits between the first-failure points of the frames (bisected on the oracle)
    so that every frame of utterance 0 and the frames before the named one solve."""
    from pytorchwavenetvocoder_b200.utils import mcep as M
    rng = np.random.RandomState(31)
    xs = [np.int16(_speechlike(rng, n)) for n in (1024 + 160, 1024 + 239, 1024 + 165)]
    fb = [[_first_failure(f, 25, 0.41, 1e-6) for f in MO.frames(x, 1024, 80)] for x in xs]
    flat = [(b, u, t) for u, bs in enumerate(fb) for t, b in enumerate(bs)]
    pick = None
    for lo, hi in zip(sorted(b for b, _, _ in flat), sorted(b for b, _, _ in flat)[1:]):
        md = np.sqrt(lo * hi)
        if hi / lo - 1 < 1e-5:
            continue
        failing = [(u, t) for b, u, t in flat if b < md]
        if failing and failing[0][0] >= 1 and failing[0][1] >= 1:
            pick = md, failing[0]
            break
    assert pick is not None, fb
    md, (u, t) = pick
    j = -MO.mcep(MO.frames(xs[u], 1024, 80)[t], 25, 0.41, min_det=md)[1]
    assert j >= 1
    monkeypatch.setattr(M, "MIN_DET", md)
    with pytest.raises(M.McepSolveError) as e:
        M.mcep_batch(xs, FS, 1024, 80, 25, 0.41)
    print("min_det %.6g: %s" % (md, e.value))
    assert "frame %d of utterance %d failed at iteration %d " % (t, u, j) in str(e.value)


# ----------------------------------------------------------------------------------------- frame-to-utterance map
@pytest.mark.parametrize("n_utts", [1, 2, 3, 257])
@pytest.mark.parametrize("cutoff", [0, 70])
def test_many_utterances_match_each_alone(n_utts, cutoff):
    """single-frame utterances (length fftl) first, last and every third; each utterance's rows and counts equal, bit
    for bit, running it alone; four utterances against the oracle"""
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    rng = np.random.RandomState(60 + n_utts + cutoff)
    lens = [1024 if i % 3 == 0 or i == n_utts - 1 else 1024 + 80 * int(rng.randint(1, 9)) + int(rng.randint(0, 80))
            for i in range(n_utts)]
    xs = [np.int16(_speechlike(rng, n)) for n in lens]
    feats, iters = mcep_batch(xs, FS, 1024, 80, 25, 0.41, highpass_cutoff=cutoff, return_iters=True)
    for u, x in enumerate(xs):
        f1, i1 = mcep_batch([x], FS, 1024, 80, 25, 0.41, highpass_cutoff=cutoff, return_iters=True)
        same = feats[u].view(np.uint32) == f1[0].view(np.uint32)
        if not same.all():
            t, m = np.argwhere(~same)[0]
            raise AssertionError("%d utterances cutoff %d: utterance %d (length %d) frame %d coefficient %d: %r in the "
                                 "batch, %r alone" % (n_utts, cutoff, u, len(x), t, m, feats[u][t, m], f1[0][t, m]))
        assert np.array_equal(iters[u], i1[0]), (n_utts, cutoff, u, iters[u], i1[0])
    which = sorted({0, n_utts // 2, max(0, n_utts - 2), n_utts - 1})
    _check(xs, FS, 1024, 80, 25, 0.41, cutoff, which=which,
           label="%d utterances cutoff %d (%d frames)" % (n_utts, cutoff, sum(len(f) for f in feats)))
