# -*- coding: utf-8 -*-
"""Mel-spectrogram features on the GPU (DESIGN.md §6 row f5): host side of ``wnb_melspc_lowcut`` and ``wnb_melspc``.

Mirrors the reference's ``melspectrogram_extract`` (bin/feature_extract.py): the 255-tap low-cut FIR
(``firwin(255, cutoff / (fs // 2), pass_zero=False)`` applied with ``lfilter``), then
``librosa.feature.melspectrogram(x / 32768, fs, n_fft=fftl, hop_length=hop, n_mels, fmin, fmax, power=1.0)`` with the
semantics of librosa 0.6.2-0.9 (``center=True`` reflect padding, periodic Hann window, Slaney mel filterbank stored as
float32) and ``np.float32(np.log10(np.maximum(1e-10, mspc.T)))``.  librosa is not needed: its filterbank is restated
here, and the window and FIR taps come from scipy, the functions the reference calls.  A batch of utterances is one
launch per stage (csrc/melspc.cu), float64 throughout with one float32 rounding at the end; there is no CPU fallback.
``MelspcStream`` extracts the same features from signals that arrive in chunks (row f7, csrc/melspc_stream.cu),
bit-identical to ``melspc_batch`` of each whole signal."""
import ctypes
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
    out, y16, off, foff = melspc_batch_device(signals, fs, fftl, hop, n_mels, fmin=fmin, fmax=fmax,
                                              highpass_cutoff=highpass_cutoff, filtered_int16=filtered_int16,
                                              device=device)
    with torch.cuda.device(out.device):
        feats = out.cpu().numpy()
        wavs = y16.cpu().numpy() if y16 is not None else None
    feats = [feats[foff[i]:foff[i + 1]] for i in range(len(signals))]
    if filtered_int16:
        return feats, [wavs[off[i]:off[i + 1]] for i in range(len(signals))]
    return feats


def melspc_batch_device(signals, fs, fftl, hop, n_mels, fmin=None, fmax=None, highpass_cutoff=0, filtered_int16=False,
                        device=None):
    """``melspc_batch`` with its results left on the device: (frames, filtered int16 wavs or None, sample offsets,
    frame offsets).  frames is one float32 CUDA tensor (total frames, n_mels) and the filtered wavs one int16 CUDA
    tensor (total samples,); utterance i owns rows ``frame_offsets[i]:frame_offsets[i + 1]`` and samples
    ``offsets[i]:offsets[i + 1]`` (host int64 arrays).  The work is queued on the current stream, not synchronised."""
    if len(signals) == 0:
        raise ValueError("melspc: no signals")
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
    return out, y16, off, foff


# ---- streaming (DESIGN.md §6 row f7) --------------------------------------------------------------------------------
MELSPC_MAX_STREAM_SEGMENTS = 1024   # WNB_MELSPC_MAX_STREAM_SEGMENTS (include/wnb200.h): keys per MelspcStream.push call
SEG_FIELDS = 11                     # WNB_MELSPC_SEG_FIELDS and the column order of include/wnb200.h
(SEG_SLOT, SEG_FLAGS, SEG_X_OFF, SEG_X_LEN, SEG_N_BEFORE, SEG_CARRY0, SEG_SCRATCH, SEG_R0, SEG_R1, SEG_OUT_ROW,
 SEG_CARRY1) = range(SEG_FIELDS)
SEG_NEW, SEG_STORE = 1, 2


def melspc_frames_ready(n, fftl, hop):
    """Frames of a centred STFT (reflect padding, ``half = fftl // 2``) that no later sample and no end position can
    change once a signal has had ``n`` samples: frame t reads ``[t hop - half, t hop + half)``, which lies in the known
    samples and, for t hop >= half is not needed, reflects about index 0 only, once ``t hop + half <= n``."""
    half = int(fftl) // 2
    return 0 if n <= half else (int(n) - half) // int(hop) + 1


def melspc_carry_start(n, fftl, hop):
    """First filtered sample the frames still pending after ``n`` samples can read, whatever the signal's final length:
    the next frame's first sample ``ready(n) hop - half``, or, if the signal ends now, the earliest sample the last
    frames reach by reflection about the end, ``n - 1 - half``.  Fewer than ``fftl`` samples are kept from here."""
    half = int(fftl) // 2
    return max(0, min(melspc_frames_ready(n, fftl, hop) * int(hop) - half, int(n) - 1 - half))


def melspc_stream_plan(segments, fftl, hop, n_taps):
    """The segment table of one ``wnb_melspc_stream`` call, from host counts only (a pure function: the numpy executor
    of tests/test_melspc_stream_host.py runs the same table on the CPU).

    segments: (slot, samples before this chunk, chunk length, key ends now) per key.  A key with no samples before
    this chunk is new: zero history and no carry, whatever its slot held.  Returns (table (n, SEG_FIELDS) int64,
    frames written, scratch doubles).  A key that ends without a sample raises ValueError."""
    hist = max(int(n_taps) - 1, 0)
    tab = np.zeros((len(segments), SEG_FIELDS), dtype=np.int64)
    x_off = rows = scratch = 0
    for u, (slot, n0, m, final) in enumerate(segments):
        n1 = n0 + m
        if final and n1 == 0:
            raise ValueError("melspc stream: a signal needs at least one sample")
        r0 = melspc_frames_ready(n0, fftl, hop)
        r1 = n_frames(n1, hop) if final else melspc_frames_ready(n1, fftl, hop)
        cs0 = melspc_carry_start(n0, fftl, hop)
        store = not final and m > 0
        flags = (SEG_NEW if n0 == 0 else 0) | (SEG_STORE if store else 0)
        tab[u] = (slot, flags, x_off, m, n0, cs0, scratch, r0, r1, rows, melspc_carry_start(n1, fftl, hop))
        if r1 > r0 or store:
            scratch += n0 - cs0 + m + (hist if store else 0)
        x_off += m
        rows += r1 - r0
    return tab, rows, scratch


class MelspcStream(object):
    """Log mel-spectrogram features of signals that arrive in chunks: ``push`` takes the next chunk of any number of
    signals, keyed by the caller, and returns every frame that no later sample can change.  Concatenated, the frames of
    a key equal ``melspc_batch`` of its whole signal bit for bit, whatever the chunk sizes (``wnb_melspc_stream`` keeps
    each key's FIR history and the filtered samples its pending frames still read on the device between calls).

    With ``scaler=(mean, scale)`` (float64, n_mels) the frames come back scaled as ``StandardScaler.transform`` scales
    the float32 features ``bin/decode.py`` reads, transposed to ``(n_mels, n)``: the aux chunk ``DecodePool.feed``
    takes and, stacked over rows, ``DecodeSession.step``.  ``scaler_mode`` (0 or 2, see
    ``device_loader._f32_scaler_mode``) defaults to what the installed scikit-learn does."""

    def __init__(self, fs, fftl, hop, n_mels, fmin=None, fmax=None, highpass_cutoff=0, scaler=None, scaler_mode=None,
                 device=None):
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", torch.cuda.current_device()) if dev.type == "cuda" and dev.index is None else dev
        if hop <= 0:
            raise ValueError("melspc stream: need a frame shift of at least one sample, got %d" % hop)
        self.fs, self.fftl, self.hop, self.n_mels = int(fs), int(fftl), int(hop), int(n_mels)
        self.n_taps = N_TAPS if highpass_cutoff else 0
        self.state_doubles = int(load().wnb_melspc_stream_state_doubles(self.fftl, self.n_taps))
        if self.state_doubles == 0:
            raise ValueError("melspc stream: fftl %d is not supported (powers of two from 64 to 4096)" % fftl)
        basis, lo, hi = mel_filterbank(fs, fftl, n_mels, 0 if fmin is None else fmin, fs // 2 if fmax is None else fmax)
        d = self.device
        self._taps = torch.from_numpy(lowcut_taps(fs, highpass_cutoff)).to(d) if highpass_cutoff else None
        self._window = torch.from_numpy(hann_window(fftl)).to(d)
        self._tw = torch.from_numpy(np.array(fft_twiddles(self.fftl))).to(d)
        self._mel = torch.from_numpy(np.array(basis)).to(d)
        self._lo, self._hi = torch.from_numpy(np.array(lo)).to(d), torch.from_numpy(np.array(hi)).to(d)
        self._mean = self._scale = None
        self.scaler_mode = 0
        if scaler is not None:
            mean, scale = (np.ascontiguousarray(a, dtype=np.float64) for a in scaler)
            if mean.shape != (self.n_mels,) or scale.shape != (self.n_mels,):
                raise ValueError("melspc stream: scaler mean and scale should have shape (%d,)" % self.n_mels)
            if scaler_mode is None:
                from .device_loader import _f32_scaler_mode
                scaler_mode = _f32_scaler_mode()
            if scaler_mode not in (0, 2):
                raise ValueError("melspc stream: scaler_mode should be 0 or 2, got %r" % (scaler_mode,))
            self.scaler_mode = int(scaler_mode)
            self._mean, self._scale = torch.from_numpy(mean).to(d), torch.from_numpy(scale).to(d)
        self._states = torch.empty(0, self.state_doubles, dtype=torch.float64, device=d)
        self._slots = {}       # key -> state slot
        self._count = {}       # key -> samples pushed so far
        self._free = []        # slots of closed keys
        self._used = 0         # slots handed out so far (the table may hold more)

    def slot(self, key):
        """The state slot of ``key``, or None when the key is not open."""
        return self._slots.get(key)

    def samples(self, key):
        """Samples pushed for ``key`` so far (None when the key is not open)."""
        return self._count.get(key)

    def push(self, chunks, final=()):
        """``{key: 1-D int16 or float64 CUDA tensor}`` (one dtype per call, int16 units) -> ``{key: frames}`` for every
        key in ``chunks`` or ``final``: float32 ``(n, n_mels)`` rows, or with a scaler the scaled ``(n_mels, n)`` aux.
        Keys in ``final`` end with this call (their chunk may be left out or empty): their remaining frames come back
        and their slot is freed.  A new key starts from zero state.  Two library launches, none when no key has samples
        or frames; the host is not synchronised."""
        final = set(final)
        keys = list(chunks) + [k for k in final if k not in chunks]
        if not keys:
            return {}
        if len(keys) > MELSPC_MAX_STREAM_SEGMENTS:
            raise ValueError("melspc stream: at most %d keys per call" % MELSPC_MAX_STREAM_SEGMENTS)
        xs = [chunks[k] for k in keys if k in chunks]
        dt = xs[0].dtype if xs else torch.int16
        if dt not in (torch.int16, torch.float64) or any(x.dtype != dt for x in xs):
            raise ValueError("melspc stream: chunks should all be int16 or all float64")
        if any(x.dim() != 1 or x.device != self.device for x in xs):
            raise ValueError("melspc stream: chunks should be 1-D tensors on %s" % self.device)
        for k in keys:
            if k in final and self._count.get(k, 0) + (chunks[k].numel() if k in chunks else 0) == 0:
                raise ValueError("melspc stream: key %r ends without a sample" % (k,))
        for k in keys:
            if k not in self._slots:
                self._open(k)
        lens = [chunks[k].numel() if k in chunks else 0 for k in keys]
        tab, rows, scratch = melspc_stream_plan([(self._slots[k], self._count[k], m, k in final)
                                                 for k, m in zip(keys, lens)], self.fftl, self.hop, self.n_taps)
        d = self.device
        out = torch.empty(rows, self.n_mels, dtype=torch.float32, device=d)
        aux = torch.empty(rows * self.n_mels, dtype=torch.float32, device=d) if self._mean is not None else None
        if rows > 0 or (tab[:, SEG_FLAGS] & SEG_STORE).any():
            x = torch.cat([chunks[k] for k in keys if k in chunks]) if sum(lens) > 0 else None
            xp = ptr(x)   # raises for CPU tensors: there is no CPU fallback
            with torch.cuda.device(d):
                host = torch.from_numpy(tab)
                segs = host.pin_memory().to(d, non_blocking=True)
                buf = torch.empty(max(scratch, 1), dtype=torch.float64, device=d)
                check(load().wnb_melspc_stream(
                    xp, 1 if dt == torch.int16 else 0, len(keys), tab.ctypes.data_as(ctypes.c_void_p), ptr(segs),
                    rows, self.fftl, self.hop, ptr(self._taps), self.n_taps, ptr(self._window), ptr(self._tw),
                    ptr(self._mel), ptr(self._lo), ptr(self._hi), self.n_mels, ptr(self._states),
                    self._states.size(0), ptr(buf), max(scratch, 1), ptr(out), ptr(self._mean), ptr(self._scale),
                    self.scaler_mode, ptr(aux), stream()), "melspc_stream")
        res = {}
        for u, (k, m) in enumerate(zip(keys, lens)):
            row, nf = int(tab[u, SEG_OUT_ROW]), int(tab[u, SEG_R1] - tab[u, SEG_R0])
            if aux is not None:
                res[k] = aux[row * self.n_mels:(row + nf) * self.n_mels].view(self.n_mels, nf)
            else:
                res[k] = out[row:row + nf]
            self._count[k] += m
        for k in final:
            self.close(k)
        return res

    def close(self, key):
        """Forget ``key`` without output; its slot goes to the next new key (which starts from zero state)."""
        s = self._slots.pop(key, None)
        if s is None:
            raise KeyError("melspc stream: unknown key %r" % (key,))
        del self._count[key]
        self._free.append(s)

    def _open(self, key):
        if self._free:
            s = min(self._free)
            self._free.remove(s)
        else:
            s, self._used = self._used, self._used + 1
            if s == self._states.size(0):   # grow the table; a new key's slot is written before it is read
                grown = torch.empty(max(2 * s, 64), self.state_doubles, dtype=torch.float64, device=self.device)
                grown[:s] = self._states
                self._states = grown
        self._slots[key] = s
        self._count[key] = 0
