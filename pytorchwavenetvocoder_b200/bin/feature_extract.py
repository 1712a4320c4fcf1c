#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""Feature extraction CLI (drop-in for reference wavenet_vocoder/bin/feature_extract.py: same flags, same
``hdf5dir/<name>.h5`` files and the same filtered int16 wavs in ``wavdir``) for ``--feature_type melspc`` (``/melspc``:
the low-cut filter and the log mel-spectrogram) and ``--feature_type mcep`` (``/mcep``: the low-cut filter and the STFT
mel-cepstra the noise-shaping recipes average), on the GPU: the wav list is processed in batches of ``--batch_size``
files, one kernel launch per stage per batch, instead of ``--n_jobs`` CPU processes (``--n_jobs`` is accepted and
ignored).  librosa and pysptk are not needed.  ``world`` (sprocket's WORLD analysis) is not provided: it exits with an
error that names the reference script.  Both feature types append to an existing feature file, so the recipes' mcep
pass adds ``/mcep`` beside ``/melspc``.  Stated deviations (DESIGN.md §6 f5, f6): ``--fmin ""`` / ``--fmax ""`` (what
the melspc recipes pass) mean "not given" instead of an argparse error; the features are computed in float64
throughout, as librosa 0.9 does (0.6-0.8 multiply the mel basis in float32); a wav shorter than ``--fftl`` has no mcep
frames: the CLI checks every wav's length first and exits 1 naming the short files before it writes anything (the
reference's worker dies in ``np.stack([])``).  Without h5py the features go to ``<name>.npz`` with the same keys, which
every reader here accepts."""
import argparse
import logging
import os
import sys

import numpy as np

from pytorchwavenetvocoder_b200.utils import find_files, read_txt, read_wav_int16, write_hdf5, write_wav_int16
from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch, shift_length


def _strtobool(v):
    v = str(v).lower()
    if v in ("y", "yes", "t", "true", "on", "1"):
        return 1
    if v in ("n", "no", "f", "false", "off", "0"):
        return 0
    raise ValueError("invalid truth value %r" % (v,))


def _optional_int(v):
    """``type=int`` for ``nargs="?"`` flags, with an empty string meaning "not given" (the recipes pass ``--fmin ""``)."""
    return None if v is None or str(v).strip() == "" else int(v)


def _feature_file(hdf5dir, wav_name, ext):
    return hdf5dir + "/" + os.path.basename(wav_name).replace(".wav", ext)


def _have_h5py():
    try:
        import h5py  # noqa: F401
        return True
    except ImportError:
        return False


def _feature_ext():
    if _have_h5py():
        return ".h5"
    logging.warning("h5py is not installed: features are written as <name>.npz with the same keys.")
    return ".npz"


def _read_batch(names, i0, n_all, args):
    xs = []
    for i, wav_name in enumerate(names):
        logging.info("now processing %s (%d/%d)" % (wav_name, i0 + i + 1, n_all))
        fs, x = read_wav_int16(wav_name)
        if x.dtype != np.int16:
            logging.warning("wav file format is not 16 bit PCM.")
        if not fs == args.fs:
            logging.error("sampling frequency is not matched.")
            sys.exit(1)
        xs.append(x)
    if not all(x.dtype == np.int16 for x in xs):
        xs = [np.array(x, dtype=np.float64) for x in xs]
    return xs


def melspectrogram_extract(wav_list, args):
    """EXTRACT MEL SPECTROGRAM (reference feature_extract.py:199-237), ``--batch_size`` files per launch."""
    ext = _feature_ext()
    save_wav = args.highpass_cutoff != 0 and args.save_wav
    bs = max(int(args.batch_size), 1)
    for i0 in range(0, len(wav_list), bs):
        names = wav_list[i0:i0 + bs]
        xs = _read_batch(names, i0, len(wav_list), args)
        out = melspc_batch(xs, args.fs, args.fftl, shift_length(args.shiftms, args.fs), args.mspc_dim, fmin=args.fmin,
                           fmax=args.fmax, highpass_cutoff=args.highpass_cutoff, filtered_int16=save_wav)
        feats, wavs = out if save_wav else (out, None)
        for j, wav_name in enumerate(names):
            write_hdf5(_feature_file(args.hdf5dir, wav_name, ext), "/melspc", feats[j])
            if save_wav:
                write_wav_int16(args.wavdir + "/" + os.path.basename(wav_name), args.fs, wavs[j])


def _n_samples(wav_name):
    """Sample count of a wav file without reading its samples (scipy's memory map; the stdlib header otherwise)."""
    try:
        from scipy.io import wavfile
        return len(wavfile.read(wav_name, mmap=True)[1])
    except ImportError:
        import wave
        with wave.open(wav_name, "rb") as w:
            return w.getnframes()


def check_mcep_lengths(wav_list, fftl):
    """Log every wav shorter than fftl (it has no mcep frames) and return whether all are long enough, so the CLI can
    stop before it writes anything."""
    ok = True
    for wav_name in wav_list:
        n = _n_samples(wav_name)
        if n < fftl:
            logging.error("%s has %d samples, fewer than fftl = %d, so it has no mcep frames; nothing was written (the "
                          "original project's wavenet_vocoder/bin/feature_extract.py stops on it too, when stft_mcep "
                          "stacks an empty list of pysptk.mcep frames)." % (wav_name, n, fftl))
            ok = False
    return ok


def mcep_extract(wav_list, args):
    """EXTRACT MCEP (reference feature_extract.py:116-148), ``--batch_size`` files per launch."""
    ext = _feature_ext()
    save_wav = args.highpass_cutoff != 0 and args.save_wav
    bs = max(int(args.batch_size), 1)
    for i0 in range(0, len(wav_list), bs):
        names = wav_list[i0:i0 + bs]
        xs = _read_batch(names, i0, len(wav_list), args)
        out = mcep_batch(xs, args.fs, args.fftl, shift_length(args.shiftms, args.fs), args.mcep_dim, args.mcep_alpha,
                         highpass_cutoff=args.highpass_cutoff, filtered_int16=save_wav)
        feats, wavs = out if save_wav else (out, None)
        for j, wav_name in enumerate(names):
            write_hdf5(_feature_file(args.hdf5dir, wav_name, ext), "/mcep", feats[j])
            if save_wav:
                write_wav_int16(args.wavdir + "/" + os.path.basename(wav_name), args.fs, wavs[j])


def get_parser():
    """Flags of reference feature_extract.py:241-300 (+ --batch_size)."""
    parser = argparse.ArgumentParser(description="making feature file argsurations.")
    parser.add_argument("--waveforms", default=None, help="directory or list of filename of input wavfile")
    parser.add_argument("--hdf5dir", default=None, help="directory to save hdf5")
    parser.add_argument("--wavdir", default=None, help="directory to save of preprocessed wav file")
    parser.add_argument("--fs", default=16000, type=int, help="Sampling frequency")
    parser.add_argument("--shiftms", default=5, type=float, help="Frame shift in msec")
    parser.add_argument("--feature_type", default="world", choices=["world", "melspc", "mcep"], type=str,
                        help="feature type")
    parser.add_argument("--mspc_dim", default=80, type=int, help="Dimension of mel spectrogram")
    parser.add_argument("--minf0", default=40, type=int, help="minimum f0 for world analysis")
    parser.add_argument("--maxf0", default=400, type=int, help="maximum f0 for world analysis")
    parser.add_argument("--fmin", default=None, nargs="?", type=_optional_int,
                        help="minimum frequency for melspc (empty: not given)")
    parser.add_argument("--fmax", default=None, nargs="?", type=_optional_int,
                        help="maximum frequency for melspc (empty: not given)")
    parser.add_argument("--mcep_dim", default=24, type=int, help="Dimension of mel cepstrum")
    parser.add_argument("--mcep_alpha", default=0.41, type=float, help="Alpha of mel cepstrum")
    parser.add_argument("--fftl", default=1024, type=int, help="FFT length")
    parser.add_argument("--highpass_cutoff", default=70, type=int, help="Cut off frequency in lowpass filter")
    parser.add_argument("--save_wav", default=True, type=_strtobool, help="Whether to save filtered wav file")
    parser.add_argument("--n_jobs", default=10, type=int,
                        help="number of parallel jobs (accepted, unused: one GPU launch per stage and batch)")
    parser.add_argument("--batch_size", default=64, type=int, help="wav files per kernel launch")
    parser.add_argument("--verbose", default=1, type=int, help="log message level")
    return parser


def main(argv=None):
    """RUN FEATURE EXTRACTION (reference feature_extract.py:240-335)."""
    args = get_parser().parse_args(argv)
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    if args.verbose == 1:
        logging.basicConfig(level=logging.INFO, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    elif args.verbose > 1:
        logging.basicConfig(level=logging.DEBUG, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    else:
        logging.basicConfig(level=logging.WARNING, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
        logging.warning("logging is disabled.")
    for key, value in vars(args).items():
        logging.info("%s = %s" % (key, str(value)))

    if args.feature_type == "world":
        logging.error("--feature_type world is not provided by this package: use the original project's "
                      "wavenet_vocoder/bin/feature_extract.py (it needs sprocket's WORLD analysis).")
        sys.exit(1)

    if os.path.isdir(args.waveforms):
        file_list = sorted(find_files(args.waveforms, "*.wav"))
    else:
        file_list = read_txt(args.waveforms)
    logging.info("number of utterances = %d" % len(file_list))
    if args.feature_type == "mcep" and not check_mcep_lengths(file_list, args.fftl):
        sys.exit(1)

    if args.highpass_cutoff != 0 and args.save_wav and not os.path.exists(args.wavdir):
        os.makedirs(args.wavdir)
    if not os.path.exists(args.hdf5dir):
        os.makedirs(args.hdf5dir)
    if args.feature_type == "melspc":
        melspectrogram_extract(file_list, args)
    else:
        mcep_extract(file_list, args)


if __name__ == "__main__":
    main()
