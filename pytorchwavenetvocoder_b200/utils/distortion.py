# -*- coding: utf-8 -*-
"""Mel-cepstral distortion (MCD) between decoded and natural speech on the GPU (DESIGN.md §6 row f8): host side of
``wnb_mcd_aligned`` and ``wnb_mcd_dtw``.

A frame's MCD in dB is ``K * dist``, ``dist = sqrt(sum_{d>=1} (c_d - c'_d)^2)`` over the mel-cepstra without c0 and
``K = fl(10 / ln 10) * fl(sqrt 2)``.  An utterance's MCD is ``K * sum(dist) / n`` over its n frames compared index by
index (``dtw=False``: the first ``min(Tr, Td)`` frames) or over the n steps of a dynamic-time-warping path
(``dtw=True``: steps (1, 1), (1, 0) and (0, 1), ties to the diagonal, then (i-1, j), then (i, j-1)).  A corpus's MCD is
frame-weighted: ``K * sum of the sums / sum of the n``.  The sums are float64 with fixed operation orders
(include/wnb200.h), so the same pair gives the same bits alone, in any batch and run after run.  The mel-cepstra come
from ``mcep_batch`` (row f6), the recipes' analysis, so numbers are comparable from run to run."""
import collections
import math

import numpy as np
import torch

from .._lib import check, load, ptr, stream
from .mcep import mcep_batch
from .melspc import _device

K = (10.0 / math.log(10.0)) * math.sqrt(2.0)
WORKSPACE_BYTES = 1 << 30        # default DTW workspace per launch; a batch that needs more is split into launches

Mcd = collections.namedtuple("Mcd", ["mcd", "counts", "sums", "paths"])
Mcd.__doc__ = """Per utterance: ``mcd`` in dB (float64), ``counts`` (int64: frames compared, or path steps), ``sums``
(float64: the summed frame distances, without K) and ``paths`` (a list of (n, 2) int32 arrays of (reference frame,
decoded frame) steps, or None)."""


def _frames(frames, what):
    out = []
    for k, f in enumerate(frames):
        a = np.ascontiguousarray(f, dtype=np.float32)
        if a.ndim != 2 or a.shape[0] < 1:
            raise ValueError("mcd: %s utterance %d should be a non-empty (frames, D + 1) array, got shape %s"
                             % (what, k, a.shape))
        out.append(a)
    return out


def dtw_workspace_bytes(ref_len, dec_len):
    """Workspace bytes ``wnb_mcd_dtw`` uses for one pair of ``ref_len`` and ``dec_len`` frames."""
    return int(load().wnb_mcd_dtw_workspace(int(ref_len), int(dec_len)))


def launch_groups(ref_lens, dec_lens, workspace_bytes):
    """Consecutive pair ranges ``[(a, b, bytes)]`` whose DTW workspaces together fit ``workspace_bytes``; a pair that
    alone needs more runs in a launch of its own."""
    groups, a, used = [], 0, 0
    for p, (tr, td) in enumerate(zip(ref_lens, dec_lens)):
        need = dtw_workspace_bytes(tr, td)
        if p > a and used + need > workspace_bytes:
            groups.append((a, p, used))
            a, used = p, 0
        used += need
    if len(ref_lens) > a:
        groups.append((a, len(ref_lens), used))
    return groups


def mcd_batch(ref_frames, dec_frames, dtw=False, return_path=False, device=None, workspace_bytes=WORKSPACE_BYTES):
    """MCD of each pair (ref_frames[k], dec_frames[k]) of (T, D + 1) float32 mel-cepstra (c0 first, 1 <= D <= 40).

    Without ``dtw`` one launch compares the first min(Tr, Td) frames index by index.  With ``dtw`` the pairs run in as
    few launches as ``workspace_bytes`` allows (at least one pair each), and ``return_path`` also returns each path.
    Nothing is synchronised until the results are copied back at the end.  Returns ``Mcd``."""
    if len(ref_frames) != len(dec_frames):
        raise ValueError("mcd: %d reference and %d decoded utterances" % (len(ref_frames), len(dec_frames)))
    if return_path and not dtw:
        raise ValueError("mcd: paths come from DTW (dtw=True)")
    n = len(ref_frames)
    if n == 0:
        return Mcd(np.zeros(0), np.zeros(0, dtype=np.int64), np.zeros(0), [] if return_path else None)
    refs, decs = _frames(ref_frames, "reference"), _frames(dec_frames, "decoded")
    cols = {a.shape[1] for a in refs + decs}
    if len(cols) != 1:
        raise ValueError("mcd: every utterance needs the same number of coefficients, got %s" % sorted(cols))
    n_cols = cols.pop()
    ref_lens = np.array([len(a) for a in refs], dtype=np.int64)
    dec_lens = np.array([len(a) for a in decs], dtype=np.int64)
    roff = np.concatenate([[0], np.cumsum(ref_lens)]).astype(np.int64)
    doff = np.concatenate([[0], np.cumsum(dec_lens)]).astype(np.int64)
    lib = load()
    dev = _device(device)
    with torch.cuda.device(dev):
        r = torch.from_numpy(np.concatenate(refs)).to(dev)
        d = torch.from_numpy(np.concatenate(decs)).to(dev)
        roff_d, doff_d = torch.from_numpy(roff).to(dev), torch.from_numpy(doff).to(dev)
        sums = torch.empty(n, dtype=torch.float64, device=dev)
        counts = torch.empty(n, dtype=torch.int64, device=dev)
        path = None
        if not dtw:
            check(lib.wnb_mcd_aligned(ptr(r), ptr(d), n_cols, ptr(roff_d), ptr(doff_d), roff.ctypes.data,
                                      doff.ctypes.data, n, ptr(sums), ptr(counts), stream()), "mcd_aligned")
        else:
            groups = launch_groups(ref_lens, dec_lens, workspace_bytes)
            ws = torch.empty(max(g[2] for g in groups), dtype=torch.uint8, device=dev)
            if return_path:
                path = torch.empty(int(roff[-1] + doff[-1] - n), 2, dtype=torch.int32, device=dev)
            for a, b, need in groups:
                slot = int(roff[a] + doff[a] - a)
                check(lib.wnb_mcd_dtw(ptr(r), ptr(d), n_cols, ptr(roff_d[a:b + 1]), ptr(doff_d[a:b + 1]),
                                      roff[a:].ctypes.data, doff[a:].ctypes.data, b - a, ptr(ws), need,
                                      ptr(sums[a:b]), ptr(counts[a:b]), None if path is None else ptr(path[slot:]),
                                      stream()), "mcd_dtw")
        sums_h, counts_h = sums.cpu().numpy(), counts.cpu().numpy()
        path_h = path.cpu().numpy() if path is not None else None
    paths = None
    if return_path:
        slots = roff[:-1] + doff[:-1] - np.arange(n)
        paths = [path_h[slots[k]:slots[k] + counts_h[k]] for k in range(n)]
    return Mcd(K * sums_h / counts_h, counts_h, sums_h, paths)


def corpus_mcd(result):
    """(frame-weighted corpus MCD ``K * sum(sums) / sum(counts)``, mean of the per-utterance MCDs), both in dB; the
    sums are added exactly (``math.fsum``) and rounded once."""
    if len(result.counts) == 0:
        return float("nan"), float("nan")
    return (K * math.fsum(result.sums) / int(np.sum(result.counts)),
            math.fsum(result.mcd) / len(result.mcd))


def mcd_wavs(ref_wavs, dec_wavs, fs, fftl, hop, order, alpha, highpass_cutoff=0, dtw=False, return_path=False,
             device=None, workspace_bytes=WORKSPACE_BYTES):
    """MCD of each pair of wavs (int16 samples, or float64 in int16 units): ``mcep_batch`` of each list with the given
    analysis (each wav at least ``fftl`` samples), then ``mcd_batch``."""
    ref = mcep_batch(ref_wavs, fs, fftl, hop, order, alpha, highpass_cutoff=highpass_cutoff, device=device)
    dec = mcep_batch(dec_wavs, fs, fftl, hop, order, alpha, highpass_cutoff=highpass_cutoff, device=device)
    return mcd_batch(ref, dec, dtw=dtw, return_path=return_path, device=device, workspace_bytes=workspace_bytes)
