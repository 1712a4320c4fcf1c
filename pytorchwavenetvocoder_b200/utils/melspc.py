# -*- coding: utf-8 -*-
"""Mel-spectrogram features on the GPU (DESIGN.md §6 row f5): host side of ``wnb_melspc_lowcut`` and ``wnb_melspc``.

Mirrors the reference's ``melspectrogram_extract`` (bin/feature_extract.py): the 255-tap low-cut FIR
(``firwin(255, cutoff / (fs // 2), pass_zero=False)`` applied with ``lfilter``), then
``librosa.feature.melspectrogram(x / 32768, fs, n_fft=fftl, hop_length=hop, n_mels, fmin, fmax, power=1.0)`` with the
semantics of librosa 0.6.2-0.9 (``center=True`` reflect padding, periodic Hann window, Slaney mel filterbank stored as
float32) and ``np.float32(np.log10(np.maximum(1e-10, mspc.T)))``.  librosa is not needed: its filterbank is restated
here, and the window and FIR taps come from scipy, the functions the reference calls.  A batch of utterances is one
launch per stage (csrc/melspc.cu), float64 throughout with one float32 rounding at the end; there is no CPU fallback."""
import functools

import numpy as np
import torch

from .._lib import check, load, ptr, stream

N_TAPS = 255        # low_cut_filter's FIR length


def shift_length(shiftms, fs):
    """Frame shift in samples as the reference computes it: ``int(shiftms * fs * 0.001)``."""
    return int(shiftms * fs * 0.001)


def n_frames(n_samples, hop):
    """Frames of a centred STFT of ``n_samples`` samples: ``1 + n_samples // hop``."""
    return 1 + int(n_samples) // int(hop)


# ---- librosa 0.6.2-0.9's Slaney mel scale (htk=False) and filterbank ------------------------------------------------
_F_SP = 200.0 / 3
_MIN_LOG_HZ = 1000.0
_MIN_LOG_MEL = _MIN_LOG_HZ / _F_SP
_LOGSTEP = np.log(6.4) / 27.0


def hz_to_mel(frequencies):
    """Slaney mel of ``frequencies`` (Hz): linear, 200/3 Hz per mel, below 1 kHz; logarithmic with step log(6.4)/27
    above."""
    f = np.atleast_1d(np.asarray(frequencies, dtype=np.float64))
    mels = f / _F_SP
    log_t = f >= _MIN_LOG_HZ
    mels[log_t] = _MIN_LOG_MEL + np.log(f[log_t] / _MIN_LOG_HZ) / _LOGSTEP
    return mels if np.ndim(frequencies) else mels[0]


def mel_to_hz(mels):
    """Inverse of ``hz_to_mel``."""
    m = np.atleast_1d(np.asarray(mels, dtype=np.float64))
    freqs = _F_SP * m
    log_t = m >= _MIN_LOG_MEL
    freqs[log_t] = _MIN_LOG_HZ * np.exp(_LOGSTEP * (m[log_t] - _MIN_LOG_MEL))
    return freqs if np.ndim(mels) else freqs[0]


@functools.lru_cache(maxsize=16)
def _mel_tables(fs, fftl, n_mels, fmin, fmax):
    fftfreqs = np.linspace(0, float(fs) / 2, int(1 + fftl // 2), endpoint=True)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, len(fftfreqs)), dtype=np.float32)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]          # float32 table times float64 norm, rounded back to float32 (librosa)
    lo = np.zeros(n_mels, dtype=np.int32)
    hi = np.zeros(n_mels, dtype=np.int32)
    for i in range(n_mels):
        nz = np.flatnonzero(weights[i])
        if len(nz):
            lo[i], hi[i] = nz[0], nz[-1] + 1
    for a in (weights, lo, hi):
        a.setflags(write=False)
    return weights, lo, hi


def mel_filterbank(fs, fftl, n_mels, fmin=0.0, fmax=None):
    """``librosa.filters.mel(fs, fftl, n_mels, fmin, fmax)`` (Slaney scale and area normalisation, float32 table of
    shape (n_mels, fftl // 2 + 1)) and each filter's nonzero bins ``[lo, hi)`` (int32; 0, 0 for an all-zero filter)."""
    fmax = float(fs) / 2 if fmax is None else fmax
    return _mel_tables(int(fs), int(fftl), int(n_mels), float(fmin), float(fmax))


def lowcut_taps(fs, cutoff):
    """The reference's low-cut FIR: ``firwin(255, cutoff / (fs // 2), pass_zero=False)`` (float64)."""
    from scipy.signal import firwin
    return np.ascontiguousarray(firwin(N_TAPS, cutoff / (fs // 2), pass_zero=False), dtype=np.float64)


def hann_window(fftl):
    """``scipy.signal.get_window("hann", fftl)``: the periodic Hann window librosa's STFT uses."""
    from scipy.signal import get_window
    return np.ascontiguousarray(get_window("hann", fftl), dtype=np.float64)


@functools.lru_cache(maxsize=8)
def fft_twiddles(fftl):
    """(fftl // 2, 2) float64: (cos, -sin)(2 pi m / fftl), evaluated in extended precision and rounded once, so each
    entry is within half an ulp (plus the extended-precision error) of the exact value."""
    m = np.arange(fftl // 2, dtype=np.longdouble)
    ang = 2 * np.arccos(np.longdouble(-1)) * m / np.longdouble(fftl)
    tw = np.stack([np.cos(ang).astype(np.float64), (-np.sin(ang)).astype(np.float64)], axis=1)
    tw = np.ascontiguousarray(tw)
    tw.setflags(write=False)
    return tw


def reflect_index(i, n):
    """The index ``np.pad(x, pad, mode="reflect")`` reads for padded position ``i`` (signal index, may be negative or
    >= n) of a signal of length ``n`` >= 1; the closed form of csrc/melspc.cu ``reflect_index``."""
    i = np.asarray(i, dtype=np.int64)
    if n == 1:
        return np.zeros_like(i)
    p = 2 * (n - 1)
    j = np.mod(i, p)
    return np.where(j < n, j, p - j)


def int16_cast(y):
    """``np.int16(y)`` of float64 values as the reference's wav writer gets it on x86-64, stated without relying on
    undefined behaviour: truncation toward zero to int32 (out of range and NaN give INT_MIN), then the low 16 bits.
    csrc/melspc.cu's ``np_int16``."""
    y = np.asarray(y, dtype=np.float64)
    ok = (y > -2147483649.0) & (y < 2147483648.0)
    i32 = np.where(ok, np.trunc(np.where(ok, y, 0.0)), -2147483648.0).astype(np.int64)
    return (i32 & 0xFFFF).astype(np.uint16).view(np.int16)


def _flatten(signals):
    """(flat numpy array, is_int16, lengths, sample offsets) of a list of 1-D signals of one dtype."""
    is_i16 = all(np.asarray(s).dtype == np.int16 for s in signals)
    dt = np.int16 if is_i16 else np.float64
    lens = np.array([len(s) for s in signals], dtype=np.int64)
    if lens.min() < 1:
        raise ValueError("melspc: every signal needs at least one sample")
    off = np.zeros(len(signals) + 1, dtype=np.int64)
    off[1:] = np.cumsum(lens)
    return np.concatenate([np.asarray(s, dtype=dt) for s in signals]), is_i16, lens, off


def _lowcut(x, is_i16, offsets, lens, fs, cutoff, want_int16):
    dev = x.device
    taps = torch.from_numpy(lowcut_taps(fs, cutoff)).to(dev)
    y = torch.empty(x.numel(), dtype=torch.float64, device=dev)
    y16 = torch.empty(x.numel(), dtype=torch.int16, device=dev) if want_int16 else None
    check(load().wnb_melspc_lowcut(ptr(x), 1 if is_i16 else 0, ptr(offsets), len(lens), int(lens.max()), ptr(taps),
                                   N_TAPS, ptr(y), ptr(y16), stream()), "melspc_lowcut")
    return y, y16


def _device(device):
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def lowcut_filter_batch(signals, fs, cutoff, device=None):
    """The reference's ``low_cut_filter`` of every signal (int16 wav samples or float64, all of one dtype), one launch:
    returns the filtered float64 signals and their ``np.int16`` casts (the filtered wavs the reference saves)."""
    if len(signals) == 0:
        return [], []
    flat, is_i16, lens, off = _flatten(signals)
    dev = _device(device)
    with torch.cuda.device(dev):
        y, y16 = _lowcut(torch.from_numpy(flat).to(dev), is_i16, torch.from_numpy(off).to(dev), lens, fs, cutoff, True)
        yh, y16h = y.cpu().numpy(), y16.cpu().numpy()
    return ([yh[off[i]:off[i + 1]] for i in range(len(signals))], [y16h[off[i]:off[i + 1]] for i in range(len(signals))])


def melspc_batch(signals, fs, fftl, hop, n_mels, fmin=None, fmax=None, highpass_cutoff=0, filtered_int16=False,
                 device=None):
    """Log mel-spectrogram features of a list of 1-D signals, one launch per stage for the whole list.

    signals: int16 arrays (wav samples) or float64 arrays in int16 units, all of one dtype, each at least one sample.
    fmin / fmax: None means 0 and fs // 2, as in the reference.  highpass_cutoff != 0 applies the reference's low-cut FIR
    first.  Returns a list of float32 arrays (frames, n_mels) with frames = 1 + len // hop; with ``filtered_int16`` also
    the list of filtered int16 wavs (``np.int16`` of the filtered float64 signal), which needs a cutoff.  An fftl the
    kernels do not cover (powers of two from 64 to 4096) raises ``WnbError``."""
    if len(signals) == 0:
        return ([], []) if filtered_int16 else []
    if filtered_int16 and not highpass_cutoff:
        raise ValueError("melspc: filtered wavs need a highpass cutoff (the reference saves them only then)")
    if hop <= 0:
        raise ValueError("melspc: need a frame shift of at least one sample, got %d" % hop)
    flat, is_i16, lens, off = _flatten(signals)
    fmin = 0 if fmin is None else fmin
    fmax = fs // 2 if fmax is None else fmax
    basis, lo, hi = mel_filterbank(fs, fftl, n_mels, fmin, fmax)
    foff = np.zeros(len(signals) + 1, dtype=np.int64)
    foff[1:] = np.cumsum(1 + lens // hop)
    dev = _device(device)
    with torch.cuda.device(dev):
        x = torch.from_numpy(flat).to(dev)
        offsets = torch.from_numpy(off).to(dev)
        y16 = None
        if highpass_cutoff:
            x, y16 = _lowcut(x, is_i16, offsets, lens, fs, highpass_cutoff, filtered_int16)
            is_i16 = False
        window = torch.from_numpy(hann_window(fftl)).to(dev)
        tw = torch.from_numpy(np.array(fft_twiddles(max(int(fftl), 2)))).to(dev)   # the library checks fftl
        mel = torch.from_numpy(np.array(basis)).to(dev)
        mlo, mhi = torch.from_numpy(np.array(lo)).to(dev), torch.from_numpy(np.array(hi)).to(dev)
        frame_offsets = torch.from_numpy(foff).to(dev)
        out = torch.empty(int(foff[-1]), n_mels, dtype=torch.float32, device=dev)
        check(load().wnb_melspc(ptr(x), 1 if is_i16 else 0, ptr(offsets), ptr(frame_offsets), len(signals),
                                int(foff[-1]), int(fftl), int(hop), ptr(window), ptr(tw), ptr(mel), ptr(mlo), ptr(mhi),
                                int(n_mels), ptr(out), stream()), "melspc")
        feats = out.cpu().numpy()
        wavs = y16.cpu().numpy() if y16 is not None else None
    feats = [feats[foff[i]:foff[i + 1]] for i in range(len(signals))]
    if filtered_int16:
        return feats, [wavs[off[i]:off[i + 1]] for i in range(len(signals))]
    return feats
