# -*- coding: utf-8 -*-
"""Checker of the GPU mel-cepstra (wnb_mcep, utils/mcep.py mcep_batch) against oracle/mcep_oracle.c, frame by frame,
shared by tests/test_gpu_mcep.py and tests/test_gpu_mcep_edges.py.

The bar.  The kernel and the oracle run the same Newton iteration in float64 but evaluate its pieces differently: a
Stockham FFT against a bit-reversed one, sums over the bins with Clenshaw and a Chebyshev recurrence against SPTK's
FFTs and freqt / frqtr recursions (equal to 1e-13 inside the supported range, tests/test_mcep_range_host.py), a
different Cholesky summation order.  These rounding differences are ~ (2M)^2 eps ~ 1e-12 relative in the warped
autocorrelations r(i) (the recurrence to order 2M = 80 dominates); Newton's step divides them by the Hessian T + H, whose
condition number stays below 1e3 on speech-like frames, so the coefficients differ by at most TOL = 1e-9 (1 + |c|).
Where the iteration counts agree, each float32 coefficient must lie in [np.float32(oracle - TOL),
np.float32(oracle + TOL)]: np.float32(oracle), or its neighbour where the oracle lies within TOL of a float32 rounding
boundary.  Where they differ, the convergence test sat on its threshold: the oracle's statistic at the first iteration
the two disagree on must lie within DELTA = 1e-9 of the threshold (the statistics differ by rounding of r(0) only), and
the GPU row must pass the same bar against the oracle forced to the GPU's count.  A failed solve (count -j) must fail
on both sides, at the same iteration: its row is the one after j - 1 updates.  Each check prints how many frames took
that branch, how many coefficients needed the neighbour, the update counts and the exits of the Newton loop."""
import collections

import numpy as np

from oracle import mcep_oracle as MO

TOL = 1e-9
DELTA = 1e-9


def _speechlike(rng, n, amp=8000.0):
    """a pulse train through a drifting all-pole filter plus noise: formant-like peaks and deep valleys"""
    from scipy.signal import lfilter
    e = rng.randn(n) * 300.0
    e[::int(rng.randint(60, 140))] += amp
    y = np.zeros(n)
    for s in range(0, n, 4000):
        a1 = 1.1 + 0.3 * np.sin(s * 1e-4)             # poles inside |z| < 0.81 for a1 in [0.8, 1.4]
        seg = lfilter([1.0], [1.0, -a1, 0.75, -0.15], e[s:s + 4000])
        y[s:s + 4000] = seg / (np.abs(seg).max() + 1e-9) * amp * (0.3 + 0.7 * rng.rand())
    return y


def _allowed(got, want):
    """got (float32) lies in [np.float32(want - TOL'), np.float32(want + TOL')], TOL' = TOL (1 + |want|): it is
    np.float32(want), or a neighbour only where the oracle lies within TOL' of a float32 rounding boundary (coefficients
    much smaller than TOL', of frames with a flat spectrum, may be any float32 in the interval); returns (ok, n_other)"""
    tol = TOL * (1.0 + np.abs(want))
    exact = got == np.float32(want)
    ok = exact | ((got >= np.float32(want - tol)) & (got <= np.float32(want + tol)))
    return ok, int((ok & ~exact).sum())


def mcep_direct(xs, fftl, hop, order, alpha, miniter=2, maxiter=30, threshold=1e-3, min_det=1e-6):
    """wnb_mcep called directly with the tables of utils/mcep.py and the given min_det (mcep_batch fixes pysptk's 1e-6
    and raises on a failed solve): the per-utterance float32 rows and update counts, negative counts included."""
    import torch
    from pytorchwavenetvocoder_b200._lib import check, load, ptr, stream
    from pytorchwavenetvocoder_b200.utils import mcep as M
    from pytorchwavenetvocoder_b200.utils.melspc import _flatten, fft_twiddles
    flat, is_i16, lens, off = _flatten(xs)
    foff = np.zeros(len(xs) + 1, dtype=np.int64)
    foff[1:] = np.cumsum((lens - fftl) // hop + 1)
    dev = torch.device("cuda", torch.cuda.current_device())

    def d(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    x, offsets, frame_offsets = d(flat), d(off), d(foff)
    window, tw = d(M.hamming_window(fftl)), d(np.array(fft_twiddles(fftl)))
    cw, W = d(M.warped_cos(fftl, alpha)), d(np.array(M.init_map(fftl, order, float(alpha))))
    al = d(M.neg_alpha_powers(order, float(alpha)))
    out = torch.empty(int(foff[-1]), order + 1, dtype=torch.float32, device=dev)
    iters = torch.empty(int(foff[-1]), dtype=torch.int32, device=dev)
    check(load().wnb_mcep(ptr(x), 1 if is_i16 else 0, ptr(offsets), ptr(frame_offsets), len(xs), int(foff[-1]),
                          int(fftl), int(hop), int(order), float(alpha), ptr(window), ptr(tw), ptr(cw), ptr(W), ptr(al),
                          int(miniter), int(maxiter), float(threshold), M.EPS, float(min_det), ptr(out), ptr(iters),
                          stream()), "mcep")
    feats, its = out.cpu().numpy(), iters.cpu().numpy()
    return ([feats[foff[i]:foff[i + 1]] for i in range(len(xs))], [its[foff[i]:foff[i + 1]] for i in range(len(xs))])


def _exit(count, maxiter):
    """which exit of the Newton loop an update count comes from"""
    if count < 0:
        return "failed solve"
    if maxiter == 0:
        return "maxiter 0"
    return "maxiter" if count == maxiter else "converged"


def _check(xs, fs, fftl, hop, order, alpha, cutoff=0, which=None, stride=1, label="", miniter=2, maxiter=30,
           threshold=1e-3, min_det=None):
    """mcep_batch of the whole list against the oracle for the utterances in ``which`` (every ``stride``-th frame), with
    the given loop settings.  With ``min_det`` wnb_mcep is called directly instead (no cutoff then), so failed solves
    come back as negative counts.  Returns {update count: frames checked}."""
    from pytorchwavenetvocoder_b200.utils.mcep import MIN_DET, mcep_batch
    from pytorchwavenetvocoder_b200.utils.melspc import lowcut_filter_batch
    loop = dict(miniter=miniter, maxiter=maxiter, threshold=threshold)
    if min_det is None:
        feats, iters = mcep_batch(xs, fs, fftl, hop, order, alpha, highpass_cutoff=cutoff, return_iters=True, **loop)
        min_det = MIN_DET
    else:
        assert not cutoff, "the direct call takes no low-cut filter"
        feats, iters = mcep_direct(xs, fftl, hop, order, alpha, min_det=min_det, **loop)
    xf = lowcut_filter_batch(xs, fs, cutoff)[0] if cutoff else xs
    n_frames = n_branch = n_neigh = 0
    hist, exits = collections.Counter(), collections.Counter()
    for u in (range(len(xs)) if which is None else which):
        fr = MO.frames(xf[u], fftl, hop)
        assert feats[u].shape == (len(fr), order + 1) and feats[u].dtype == np.float32, (label, u, feats[u].shape)
        for t in range(0, len(fr), stride):
            where = "%s utterance %d (length %d) frame %d" % (label, u, len(xs[u]), t)
            want, n, st = MO.mcep(fr[t], order, alpha, min_det=min_det, **loop)
            g = int(iters[u][t])
            hist[g] += 1
            exits[_exit(g, maxiter)] += 1
            assert (g < 0) == (n < 0), "%s: GPU count %d, oracle count %d: one solve failed, the other did not" \
                % (where, g, n)
            if g != n:
                assert g >= 0, "%s: the GPU solve failed at iteration %d, the oracle's at %d" % (where, -g, -n)
                j = min(g, n) + 1
                assert abs(st[j] - threshold) <= DELTA, "%s: GPU %d updates, oracle %d, oracle statistic %r at " \
                    "iteration %d is not within %g of the threshold %g" % (where, g, n, st[j], j, DELTA, threshold)
                want = MO.mcep(fr[t], order, alpha, min_det=min_det, force_iters=g)[0]
                n_branch += 1
            ok, nn = _allowed(feats[u][t], want)
            if not ok.all():
                m = int(np.argmin(ok))
                raise AssertionError("%s coefficient %d: GPU %r, np.float32(oracle) %r (oracle64 %r, %d updates)"
                                     % (where, m, feats[u][t][m], np.float32(want[m]), want[m], g))
            n_neigh += nn
            n_frames += 1
    print("%s: %d frames checked, %d with a different iteration count, %d coefficients took the neighbour; update "
          "counts %s; exits %s" % (label, n_frames, n_branch, n_neigh, dict(sorted(hist.items())),
                                   dict(sorted(exits.items()))))
    return dict(hist)
