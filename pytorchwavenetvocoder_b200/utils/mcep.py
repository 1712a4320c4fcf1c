# -*- coding: utf-8 -*-
"""STFT mel-cepstra on the GPU (DESIGN.md §6 row f6): host side of ``wnb_mcep``.

Mirrors the reference's ``stft_mcep`` (bin/feature_extract.py): frames ``x[hop i : hop i + fftl]`` of the signal in
int16 units (no padding, no centring; ``(len - fftl) // hop + 1`` frames) times the periodic Hamming window, and
``pysptk.mcep(frame, order, alpha, eps=1e-10, etype=1)`` of every frame, written as float32.  pysptk is not needed:
SPTK's Newton-Raphson mel-cepstral analysis runs in csrc/mcep.cu, one launch for every frame of a batch of utterances,
float64 throughout with one float32 rounding at the end; there is no CPU fallback.  The optional low-cut FIR and the
int16 wavs are melspc's (``utils/melspc.py``), run the same way."""
import functools

import numpy as np
import torch

from .._lib import check, load, ptr, stream
from .melspc import _device, _flatten, _lowcut, fft_twiddles

EPS = 1e-10          # the reference's pysptk.mcep(..., eps=1e-10, etype=1)
MIN_DET = 1e-6       # pysptk's default


class McepSolveError(RuntimeError):
    """The Newton update of a frame could not be solved (a Cholesky pivot below min_det)."""


def n_frames(n_samples, fftl, hop):
    """Frames of stft_mcep: ``(len - fftl) // hop + 1``; a signal shorter than fftl has none."""
    return max(0, (int(n_samples) - int(fftl)) // int(hop) + 1)


def hamming_window(fftl):
    """``scipy.signal.get_window("hamming", fftl)``: the periodic Hamming window stft_mcep uses."""
    from scipy.signal import get_window
    return np.ascontiguousarray(get_window("hamming", fftl), dtype=np.float64)


def warped_cos(fftl, alpha):
    """cos w~_k for k = 0 .. fftl / 2: the all-pass phase w~ = w + 2 atan(alpha sin w / (1 - alpha cos w)) at
    w = 2 pi k / fftl, by cos w~ = ((1 + alpha^2) cos w - 2 alpha) / (1 + alpha^2 - 2 alpha cos w) in extended
    precision, rounded once."""
    a = np.longdouble(alpha)
    w = 2 * np.arccos(np.longdouble(-1)) * np.arange(fftl // 2 + 1, dtype=np.longdouble) / np.longdouble(fftl)
    cw = np.cos(w)
    return np.ascontiguousarray(((1 + a * a) * cw - 2 * a) / (1 + a * a - 2 * a * cw), dtype=np.float64)


def _freqt_columns(c1, m2, a):
    """SPTK freqt applied to every column of c1 ((m1 + 1) x ncol): the warped (m2 + 1) x ncol coefficients."""
    b = 1 - a * a
    g = np.zeros((m2 + 1, c1.shape[1]), dtype=c1.dtype)
    for i in range(c1.shape[0] - 1, -1, -1):
        d = g.copy()
        g[0] = c1[i] + a * d[0]
        if m2 >= 1:
            g[1] = b * d[0] + a * d[1]
        for j in range(2, m2 + 1):
            g[j] = d[j - 1] + a * (d[j] - g[j - 1])
    return g


@functools.lru_cache(maxsize=8)
def init_map(fftl, order, alpha):
    """(order + 2, fftl / 2 + 1) float64: rows 0 .. order map log P (bins 0 .. fftl / 2) to SPTK mcep's initial value
    (the real cepstrum c_n = (1/L) sum over all L bins of log P_k cos(2 pi n k / L), c[0] and c[L/2] halved, then freqt
    to the order); row order + 1 is the halved c[0], the seed of the convergence test.  Evaluated in extended
    precision, rounded once."""
    L, nb = int(fftl), int(fftl) // 2 + 1
    ld = np.longdouble
    k = np.arange(nb)
    mult = np.where((k == 0) | (k == nb - 1), 1, 2).astype(ld)
    ang = 2 * np.arccos(ld(-1)) / ld(L)
    C = np.cos(ang * np.outer(np.arange(nb), k).astype(ld)) * mult[None, :] / ld(L)
    C[0] /= 2
    C[nb - 1] /= 2
    W = np.concatenate([_freqt_columns(C, int(order), ld(alpha)), C[:1]], axis=0)
    W = np.ascontiguousarray(W, dtype=np.float64)
    W.setflags(write=False)
    return W


def neg_alpha_powers(order, alpha):
    """(-alpha)^m for m = 0 .. order, by repeated multiplication as SPTK forms them."""
    al = np.empty(order + 1, dtype=np.float64)
    al[0] = 1.0
    for i in range(1, order + 1):
        al[i] = -alpha * al[i - 1]
    return al


def mcep_batch(signals, fs, fftl, hop, order, alpha, highpass_cutoff=0, filtered_int16=False, miniter=2, maxiter=30,
               threshold=1e-3, device=None, return_iters=False):
    """STFT mel-cepstra of a list of 1-D signals, one launch for every frame of the list.

    signals: int16 arrays (wav samples) or float64 arrays in int16 units, all of one dtype, each at least fftl samples
    long (a shorter one raises ``ValueError`` naming its length: it has no frames).  highpass_cutoff != 0 applies the
    reference's low-cut FIR first (fs picks its taps).  Returns a list of float32 arrays (frames, order + 1); with
    ``filtered_int16`` also the list of filtered int16 wavs (needs a cutoff); with ``return_iters`` also the list of
    per-frame Newton update counts (int32).  A failed solve raises ``McepSolveError`` naming the utterance and the frame.
    A shape outside the kernel's range (fftl a power of two from 1024 to 4096, order <= 40, 0 <= alpha <= 0.6) raises
    ``WnbError``."""
    if len(signals) == 0:
        out = ([],) + (([],) if filtered_int16 else ()) + (([],) if return_iters else ())
        return out if len(out) > 1 else []
    if filtered_int16 and not highpass_cutoff:
        raise ValueError("mcep: filtered wavs need a highpass cutoff (the reference saves them only then)")
    if hop <= 0:
        raise ValueError("mcep: need a frame shift of at least one sample, got %d" % hop)
    for i, s in enumerate(signals):
        if len(s) < fftl:
            raise ValueError("mcep: utterance %d has %d samples, fewer than fftl = %d, so it has no frames"
                             % (i, len(s), fftl))
    flat, is_i16, lens, off = _flatten(signals)
    foff = np.zeros(len(signals) + 1, dtype=np.int64)
    foff[1:] = np.cumsum((lens - fftl) // hop + 1)
    dev = _device(device)
    with torch.cuda.device(dev):
        x = torch.from_numpy(flat).to(dev)
        offsets = torch.from_numpy(off).to(dev)
        y16 = None
        if highpass_cutoff:
            x, y16 = _lowcut(x, is_i16, offsets, lens, fs, highpass_cutoff, filtered_int16)
            is_i16 = False
        # the tables of a shape the library cannot take are stand-ins: it rejects the shape before reading them
        plausible = int(fftl) >= 2 and int(fftl) & (int(fftl) - 1) == 0 and 1 <= int(order) <= 64
        m = int(order) if plausible else 1
        L = int(fftl) if plausible else 2
        window = torch.from_numpy(hamming_window(L)).to(dev)
        tw = torch.from_numpy(np.array(fft_twiddles(L))).to(dev)
        cw = torch.from_numpy(warped_cos(L, alpha)).to(dev)
        W = torch.from_numpy(np.array(init_map(L, m, float(alpha)))).to(dev)
        al = torch.from_numpy(neg_alpha_powers(m, float(alpha))).to(dev)
        frame_offsets = torch.from_numpy(foff).to(dev)
        out = torch.empty(int(foff[-1]), m + 1, dtype=torch.float32, device=dev)
        iters = torch.empty(int(foff[-1]), dtype=torch.int32, device=dev)
        check(load().wnb_mcep(ptr(x), 1 if is_i16 else 0, ptr(offsets), ptr(frame_offsets), len(signals),
                              int(foff[-1]), int(fftl), int(hop), int(order), float(alpha), ptr(window), ptr(tw),
                              ptr(cw), ptr(W), ptr(al), int(miniter), int(maxiter), float(threshold), EPS, MIN_DET,
                              ptr(out), ptr(iters), stream()), "mcep")
        feats = out.cpu().numpy()
        its = iters.cpu().numpy()
        wavs = y16.cpu().numpy() if y16 is not None else None
    bad = np.flatnonzero(its < 0)
    if len(bad):
        f = int(bad[0])
        u = int(np.searchsorted(foff, f, side="right") - 1)
        raise McepSolveError("mcep: the Newton update of frame %d of utterance %d failed at iteration %d (a Cholesky "
                             "pivot below %g)" % (f - foff[u], u, -its[f], MIN_DET))
    res = ([feats[foff[i]:foff[i + 1]] for i in range(len(signals))],)
    if filtered_int16:
        res += ([wavs[off[i]:off[i + 1]] for i in range(len(signals))],)
    if return_iters:
        res += ([its[foff[i]:foff[i + 1]] for i in range(len(signals))],)
    return res if len(res) > 1 else res[0]
