# -*- coding: utf-8 -*-
"""MLSA noise shaping on the GPU (SURVEY.md 8 row f4): host side of ``wnb_mlsa_filter``.

Mirrors what the reference does through pysptk (reference bin/noise_shaping.py:28-43, 46-87): ``mc2b`` turns the scaled
average mel-cepstrum into MLSA filter coefficients, and every wav file is passed through the time-invariant MLSA filter
(``Synthesizer(MLSADF(order, alpha), hopsize).synthesis`` with one coefficient row tiled over all frames).  Here a whole
list of utterances is filtered by ONE kernel launch (csrc/mlsa.cu); there is no CPU fallback.  ``MlsaStreamFilter``
filters signals that arrive in chunks (decode sessions and pools), bit-identical to filtering each whole signal."""
import ctypes

import numpy as np
import torch

from .._lib import check, load, ptr, stream

MLSA_MAX_STATE_SEGMENTS = 1024   # WNB_MLSA_MAX_STATE_SEGMENTS (include/wnb200.h): chunks per MlsaStreamFilter.filter call


def mc2b(mc, alpha):
    """SPTK ``mc2b`` (``pysptk.mc2b``, reference noise_shaping.py:41): b[m] = mc[m]; b[i] = mc[i] - alpha * b[i+1]."""
    mc = np.asarray(mc, dtype=np.float64)
    b = np.empty_like(mc)
    b[-1] = mc[-1]
    for i in range(len(mc) - 2, -1, -1):
        b[i] = mc[i] - alpha * b[i + 1]
    return b


def convert_mcep_to_mlsa_coef(avg_mcep, mag, alpha):
    """CONVERT AVERAGE MEL-CEPTSRUM TO MLSA FILTER COEFFICIENT (reference noise_shaping.py:28-43; like the reference the
    argument is scaled IN PLACE when it is a float64 array)."""
    avg_mcep *= mag
    avg_mcep[0] = 0.0
    coef = mc2b(avg_mcep.astype(np.float64), alpha)
    assert np.isfinite(coef).all()
    return coef


def mlsa_filter_batch(signals, coef, alpha, pd=4, out_int16=None, device=None):
    """Filter a list of 1-D signals with the time-invariant MLSA filter ``coef`` (order + 1 values from ``mc2b``; pass
    ``-coef`` for the inverse filter, reference noise_shaping.py:55-56).

    signals: list of int16 arrays (wav samples; converted like ``np.float64(x)``) or float64 arrays, all of one dtype.
    Returns a list of arrays of the same lengths: int16 (``np.int16(y)``, truncation toward zero, the reference's wav
    output) when the input is int16 or ``out_int16`` is True, float64 otherwise.  One launch for the whole list; every
    utterance starts from a zero filter state."""
    if len(signals) == 0:
        return []
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    is_i16 = all(np.asarray(s).dtype == np.int16 for s in signals)
    if out_int16 is None:
        out_int16 = is_i16
    dt = np.int16 if is_i16 else np.float64
    lens = [len(s) for s in signals]
    off = np.zeros(len(signals) + 1, dtype=np.int64)
    off[1:] = np.cumsum(lens)
    flat = np.concatenate([np.asarray(s, dtype=dt) for s in signals]) if off[-1] > 0 else np.zeros(0, dtype=dt)
    if off[-1] == 0:
        return [np.zeros(0, dtype=np.int16 if out_int16 else np.float64) for _ in signals]
    with torch.cuda.device(dev):
        y = mlsa_filter_device(torch.from_numpy(flat).to(dev), off, coef, alpha, pd=pd, out_int16=out_int16)
        yh = y.cpu().numpy()
    return [yh[off[i]:off[i + 1]] for i in range(len(signals))]


def mlsa_filter_device(x, offsets, coef, alpha, pd=4, out_int16=False):
    """``mlsa_filter_batch`` of signals already on the device: x is one int16 or float64 CUDA tensor holding the signals
    back to back, signal i at ``offsets[i]:offsets[i + 1]`` (host int64 array, offsets[-1] == x.numel() > 0).  Returns
    the filtered CUDA tensor of the same length (int16 with ``out_int16``, float64 otherwise), queued on the current
    stream."""
    coef = np.ascontiguousarray(coef, dtype=np.float64)
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    if x.dtype not in (torch.int16, torch.float64) or x.dim() != 1 or off[-1] != x.numel() or x.numel() == 0:
        raise ValueError("MLSA filter: x should be a non-empty 1-D int16 or float64 tensor of offsets[-1] samples")
    with torch.cuda.device(x.device):
        d_off = torch.from_numpy(off).to(x.device)
        b = torch.from_numpy(coef).to(x.device)
        y = torch.empty(x.numel(), dtype=torch.int16 if out_int16 else torch.float64, device=x.device)
        check(load().wnb_mlsa_filter(ptr(x), 1 if x.dtype == torch.int16 else 0, ptr(d_off), len(off) - 1, ptr(b),
                                     len(coef) - 1, float(alpha), int(pd), float(np.exp(coef[0])), ptr(y),
                                     1 if out_int16 else 0, stream()), "mlsa_filter")
    return y


class MlsaStreamFilter(object):
    """The time-invariant MLSA filter ``coef`` applied to signals that arrive in chunks: ``filter`` takes the next chunk
    of any number of signals, keyed by the caller, and returns their filtered chunks.  Concatenated, the chunks of a
    signal equal ``mlsa_filter_batch`` of the whole signal bit for bit, whatever the chunk sizes (``wnb_mlsa_filter_state``
    keeps each signal's filter state on the device between calls).  Pass ``coef`` as ``bin/noise_shaping.py`` does:
    ``+coef`` restores a noise-weighted signal, ``-coef`` applies the weighting.

    For a decode session the keys are row indices and the chunks ``pcm[b, :last_counts[b]]``; for a decode pool the keys
    are the stream ids ``DecodePool.step_pcm16`` returns."""

    def __init__(self, coef, alpha, pd=4, device=None):
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", torch.cuda.current_device()) if dev.type == "cuda" and dev.index is None else dev
        coef = np.ascontiguousarray(coef, dtype=np.float64)
        self.order, self.alpha, self.pd = len(coef) - 1, float(alpha), int(pd)
        self.gain = float(np.exp(coef[0]))
        self.state_doubles = int(load().wnb_mlsa_state_doubles(self.order, self.pd))
        if self.state_doubles == 0:
            raise ValueError("MLSA filter: need 2 <= order <= 255 and pd 4 or 5, got order %d, pd %d" % (self.order, pd))
        self._coef = torch.from_numpy(coef).to(self.device)
        self._states = torch.empty(0, self.state_doubles, dtype=torch.float64, device=self.device)
        self._slots = {}       # key -> state slot
        self._free = []        # slots of closed keys
        self._used = 0         # slots handed out so far (the table may hold more)
        self._fresh = set()    # keys whose slot has not been through a launch yet: their next launch starts from zero

    def slot(self, key):
        """The state slot of ``key``, or None when the key is not open."""
        return self._slots.get(key)

    def filter(self, chunks):
        """``{key: 1-D int16 or float64 CUDA tensor}`` -> ``{key: filtered chunk}`` of the same dtype and length (int16
        out by truncation toward zero, like ``np.int16(y)``).  A new key starts from a zero state.  One library launch
        for the whole dict, none when every chunk is empty; the host is not synchronised."""
        if not chunks:
            return {}
        keys = list(chunks)
        xs = [chunks[k] for k in keys]
        dt = xs[0].dtype
        if dt not in (torch.int16, torch.float64) or any(x.dtype != dt for x in xs):
            raise ValueError("MLSA filter: chunks should all be int16 or all float64")
        if any(x.dim() != 1 or x.device != self.device for x in xs):
            raise ValueError("MLSA filter: chunks should be 1-D tensors on %s" % self.device)
        if len(keys) > MLSA_MAX_STATE_SEGMENTS:
            raise ValueError("MLSA filter: at most %d chunks per call" % MLSA_MAX_STATE_SEGMENTS)
        for k in keys:
            if k not in self._slots:
                self._open(k)
        off = np.zeros(len(keys) + 1, dtype=np.int64)
        off[1:] = np.cumsum([x.numel() for x in xs])
        y = torch.empty(int(off[-1]), dtype=dt, device=self.device)
        if off[-1] > 0:
            flat = torch.cat(xs) if len(xs) > 1 else xs[0].contiguous()
            xp = ptr(flat)   # raises for CPU tensors: there is no CPU fallback
            slots = (ctypes.c_int32 * len(keys))(*[self._slots[k] for k in keys])
            zero = (ctypes.c_int32 * len(keys))(*[int(k in self._fresh) for k in keys])
            i16 = 1 if dt == torch.int16 else 0
            with torch.cuda.device(self.device):
                offsets = torch.from_numpy(off).pin_memory().to(self.device, non_blocking=True)
                check(load().wnb_mlsa_filter_state(xp, i16, ptr(offsets), len(keys), ptr(self._coef), self.order,
                                                   self.alpha, self.pd, self.gain, ptr(y), i16, ptr(self._states),
                                                   self._states.size(0), slots, zero, stream()),
                      "mlsa_filter_state")
            self._fresh.difference_update(k for k, x in zip(keys, xs) if x.numel() > 0)   # an empty chunk stores nothing
        return {k: y[off[i]:off[i + 1]] for i, k in enumerate(keys)}

    def close(self, key):
        """Forget ``key``; its slot goes to the next new key (which starts from a zero state)."""
        s = self._slots.pop(key, None)
        if s is None:
            raise KeyError("MLSA filter: unknown key %r" % (key,))
        self._fresh.discard(key)
        self._free.append(s)

    def _open(self, key):
        if self._free:
            s = min(self._free)
            self._free.remove(s)
        else:
            s, self._used = self._used, self._used + 1
            if s == self._states.size(0):   # grow the table; a new slot is written (zero start) before it is read
                grown = torch.empty(max(2 * s, 64), self.state_doubles, dtype=torch.float64, device=self.device)
                grown[:s] = self._states
                self._states = grown
        self._slots[key] = s
        self._fresh.add(key)
