# -*- coding: utf-8 -*-
"""A training corpus prepared on the device from wavs alone, and kept resident in HBM (DESIGN.md §6 row f9).

``prepare_corpus`` does what stages 1-3 of the ``*-melspc`` recipes write to disk, without writing anything but the
statistics:

1. ``feature_extract.py --feature_type melspc``: the low-cut filter and the mel-spectrogram of every wav
   (``melspc_batch_device``), keeping the float32 frames and the low-cut int16 waveform on the device;
2. with noise shaping, ``feature_extract.py --feature_type mcep --save_wav false`` (``mcep_batch`` of the raw wavs);
3. ``calc_stats.py`` for melspc (and mcep): ``StandardScaler.partial_fit`` of every utterance's frames in list order,
   stored as float32 as the stats file holds them;
4. with noise shaping, ``noise_shaping.py --feature_type mcep --inv true``: the MLSA coefficients of the float32 mcep
   mean, and the inverse filter over the low-cut int16 waveform (``mlsa_filter_device``).

Each utterance is trimmed as ``device_loader.load_pair_frames`` trims it in the up-sampling mode (whole frames, the
samples of the last frame or two dropped); the MLSA filter is causal, so filtering the trimmed waveform gives the kept
samples of the filtered whole wav.  The resident layout is one int16 waveform buffer and one float32 (frames, n_mels)
buffer, utterance k at sample ``offsets[k]`` and frame ``offsets[k] // U``.  ``DeviceCorpusGenerator``
(utils/device_loader.py) cuts training batches out of it."""
import logging
import time

import numpy as np
import torch

from .melspc import melspc_batch_device, shift_length
from .utils import read_wav_int16, write_hdf5

FILE_PIPELINE = ("the file pipeline: feature_extract.py (melspc, and mcep for noise shaping), calc_stats.py, "
                 "noise_shaping.py, then train.py --feats --stats")


class CorpusTooLarge(ValueError):
    """The resident corpus would take more than half of the free device memory."""


def trimmed_length(n, U):
    """(samples, frames) that ``load_pair_frames`` keeps of an utterance of ``n`` samples and its ``1 + n // U`` melspc
    frames at hop U: the frames drop the last one (two when n is a multiple of U), the samples follow the frames."""
    nf = 1 + int(n) // U
    mod_y = nf * U - int(n)                 # > 0 always
    nf = max(nf - (mod_y // U + 1), 0)
    return nf * U, nf


def resident_bytes(n_samples, U, n_mels):
    """Device bytes of the resident corpus of utterances of ``n_samples`` samples: int16 samples + float32 frames."""
    kept = [trimmed_length(n, U) for n in n_samples]
    return 2 * sum(s for s, _ in kept) + 4 * n_mels * sum(f for _, f in kept)


def fit_refusal(nbytes, free_bytes):
    """The refusal message when a resident corpus of ``nbytes`` exceeds half of ``free_bytes``, else None."""
    if nbytes <= free_bytes // 2:
        return None
    return ("the resident corpus needs %d bytes (%.2f GB) but half of the free device memory is %d bytes (%.2f GB); "
            "use %s" % (nbytes, nbytes / 1e9, free_bytes // 2, free_bytes / 2e9, FILE_PIPELINE))


def wav_header(path):
    """(sampling rate, samples, dtype) of a wav file without reading its samples."""
    from scipy.io import wavfile
    fs, data = wavfile.read(path, mmap=True)
    return int(fs), len(data), data.dtype


def wav_refusals(wav_list, fs, fftl):
    """Messages for every wav that the corpus cannot take: another sampling rate, not 16-bit PCM, or fewer than ``fftl``
    samples (it has no mcep frames; ``feature_extract.check_mcep_lengths``)."""
    out = []
    for w in wav_list:
        rate, n, dt = wav_header(w)
        if rate != fs:
            out.append("%s: sampling rate %d, not --fs %d" % (w, rate, fs))
        elif dt != np.int16:
            out.append("%s: %s samples, not 16-bit PCM" % (w, dt))
        elif n < fftl:
            out.append("%s has %d samples, fewer than fftl = %d, so it has no mcep frames" % (w, n, fftl))
    return out


class ResidentCorpus(object):
    """The prepared corpus: ``wave`` (int16 CUDA, total samples), ``feat`` (float32 CUDA, (total frames, n_mels)),
    ``lengths`` / ``offsets`` (host int64: kept samples and first sample of each utterance, list order), ``U``,
    ``mean`` / ``scale`` (float64 of the float32 melspc statistics), ``stats`` (every dataset of the stats file, in
    the order it is written) and ``times`` (seconds per preparation stage)."""

    def __init__(self, wave, feat, lengths, offsets, U, stats, times):
        self.wave, self.feat, self.lengths, self.offsets, self.U = wave, feat, lengths, offsets, U
        self.stats, self.times = stats, times
        self.mean = np.asarray(stats["/melspc/mean"], dtype=np.float64)
        self.scale = np.asarray(stats["/melspc/scale"], dtype=np.float64)

    def write_stats(self, path):
        """Write the statistics as ``calc_stats.py`` (and ``noise_shaping.py``) write them to ``path``."""
        for key, value in self.stats.items():
            write_hdf5(path, key, value)


def prepare_corpus(wav_list, fs=16000, shiftms=5, fftl=1024, mspc_dim=80, fmin=None, fmax=None, highpass_cutoff=70,
                   noise_shaping=False, mcep_dim=24, mcep_alpha=0.41, mag=0.5, batch_size=64, device=None):
    """Prepare the resident corpus of ``wav_list`` (in this order) on ``device`` with ``feature_extract.py``'s,
    ``noise_shaping.py``'s and their defaults' settings.  Raises ValueError for wavs ``wav_refusals`` names and
    ``CorpusTooLarge`` before anything is extracted when the corpus exceeds half of the free device memory."""
    from sklearn.preprocessing import StandardScaler
    from .mcep import mcep_batch
    from .mlsa import convert_mcep_to_mlsa_coef, mlsa_filter_device
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    U = shift_length(shiftms, fs)
    bad = wav_refusals(wav_list, fs, fftl)
    if bad:
        raise ValueError("; ".join(bad))
    n_samples = [wav_header(w)[1] for w in wav_list]
    kept = np.array([trimmed_length(n, U) for n in n_samples], dtype=np.int64).reshape(-1, 2)
    lengths = kept[:, 0].copy()
    offsets = np.zeros(len(wav_list), dtype=np.int64)
    offsets[1:] = np.cumsum(lengths)[:-1]
    refusal = fit_refusal(resident_bytes(n_samples, U, mspc_dim), torch.cuda.mem_get_info(dev)[0])
    if refusal is not None:
        raise CorpusTooLarge(refusal)
    times = dict.fromkeys(["read", "melspc", "mcep", "stats", "mlsa"], 0.0)

    def lap(key, t0):
        torch.cuda.synchronize(dev)
        t1 = time.time()
        times[key] += t1 - t0
        return t1

    with torch.cuda.device(dev):
        wave = torch.empty(int(lengths.sum()), dtype=torch.int16, device=dev)
        feat = torch.empty(int(kept[:, 1].sum()), mspc_dim, dtype=torch.float32, device=dev)
        sc_mel, sc_mcep = StandardScaler(), StandardScaler()
        bs = max(int(batch_size), 1)
        for i0 in range(0, len(wav_list), bs):
            t = time.time()
            xs = [read_wav_int16(w)[1] for w in wav_list[i0:i0 + bs]]
            t = lap("read", t)
            frames, y16, off, foff = melspc_batch_device(xs, fs, fftl, U, mspc_dim, fmin=fmin, fmax=fmax,
                                                         highpass_cutoff=highpass_cutoff,
                                                         filtered_int16=bool(highpass_cutoff), device=dev)
            if y16 is None:
                y16 = torch.from_numpy(np.concatenate(xs)).to(dev)
            for i in range(len(xs)):
                k, (n, nf) = i0 + i, kept[i0 + i]
                wave[offsets[k]:offsets[k] + n] = y16[off[i]:off[i] + n]
                feat[offsets[k] // U:offsets[k] // U + nf] = frames[foff[i]:foff[i] + nf]
            t = lap("melspc", t)
            fh = frames.cpu().numpy()
            for i in range(len(xs)):                                   # calc_stats.py, list order
                sc_mel.partial_fit(fh[foff[i]:foff[i + 1]])
            t = lap("stats", t)
            if noise_shaping:
                mc = mcep_batch(xs, fs, fftl, U, mcep_dim, mcep_alpha, highpass_cutoff=highpass_cutoff, device=dev)
                t = lap("mcep", t)
                for m in mc:
                    sc_mcep.partial_fit(m)
                t = lap("stats", t)
            del frames, y16
        stats = {"/melspc/mean": np.float32(sc_mel.mean_), "/melspc/scale": np.float32(sc_mel.scale_)}
        if noise_shaping:
            t = time.time()
            stats["/mcep/mean"] = np.float32(sc_mcep.mean_)
            stats["/mcep/scale"] = np.float32(sc_mcep.scale_)
            # noise_shaping.py: the coefficients of the stored (float32) mcep mean, applied inverted
            coef = convert_mcep_to_mlsa_coef(np.array(stats["/mcep/mean"], dtype=np.float64), mag, mcep_alpha)
            stats["/mlsa/coef"] = coef
            stats["/mlsa/alpha"] = mcep_alpha
            ends = offsets + lengths
            u0 = 0
            chunk = 1 << 28                                            # samples filtered per launch
            while u0 < len(wav_list):
                u1 = int(np.searchsorted(ends, offsets[u0] + chunk, side="right"))
                u1 = max(u1, u0 + 1)
                a, b = int(offsets[u0]), int(ends[u1 - 1])
                if b > a:
                    bounds = np.concatenate([offsets[u0:u1], ends[u1 - 1:u1]]) - a
                    wave[a:b] = mlsa_filter_device(wave[a:b], bounds, -coef, mcep_alpha, pd=4, out_int16=True)
                u0 = u1
            lap("mlsa", t)
    logging.info("resident corpus: %d utterances, %d samples, %d frames (%.2f GB); preparation %s" % (
        len(wav_list), wave.numel(), feat.size(0), (2 * wave.numel() + 4 * feat.numel()) / 1e9,
        ", ".join("%s %.2f s" % kv for kv in times.items())))
    return ResidentCorpus(wave, feat, lengths, offsets, U, stats, times)
