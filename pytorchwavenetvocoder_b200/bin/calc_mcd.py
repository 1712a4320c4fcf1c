#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""MEL-CEPSTRAL DISTORTION between decoded and natural wavs on the GPU (``utils/distortion.py``, DESIGN.md §6 row f8).

``--reference`` and ``--decoded`` are directories of wavs or lists of wav files, paired by basename.  Both sides go
through the mel-cepstral analysis of ``feature_extract.py --feature_type mcep`` (the low-cut filter, then
``mcep_batch``), ``--batch_size`` pairs per launch, and each pair is compared frame by frame: index by index by default
(copy synthesis writes sample t for natural sample t, so frames on the same grid line up), or along a DTW path with
``--dtw`` (decodes from predicted features, another sampling-rate path, a trimmed file).  ``--outfile`` gets one TSV row
per utterance (utterance id, frames compared or path steps, MCD in dB) and a ``<corpus>`` row (all frames, the
frame-weighted corpus MCD); the corpus MCD and the mean of the per-utterance MCDs are logged.

Before anything is computed, the CLI exits 1 if a file has no counterpart, a sampling rate differs from ``--fs``, a
wav is shorter than ``--fftl`` (it has no frames), or, without ``--dtw``, the frame counts of a pair differ by more
than ``--max_frame_diff``."""
import argparse
import logging
import os
import sys

import numpy as np

from pytorchwavenetvocoder_b200.utils import find_files, read_txt, read_wav_int16
from pytorchwavenetvocoder_b200.utils.mcep import n_frames
from pytorchwavenetvocoder_b200.utils.melspc import shift_length


def get_parser():
    parser = argparse.ArgumentParser(description="mel-cepstral distortion of decoded wavs against natural wavs")
    parser.add_argument("--reference", required=True, type=str, help="directory or list of natural wav files")
    parser.add_argument("--decoded", required=True, type=str, help="directory or list of decoded wav files")
    parser.add_argument("--fs", default=16000, type=int, help="Sampling frequency")
    parser.add_argument("--shiftms", default=5, type=float, help="Frame shift in msec")
    parser.add_argument("--fftl", default=1024, type=int, help="FFT length")
    parser.add_argument("--mcep_dim", default=24, type=int, help="Dimension of mel cepstrum")
    parser.add_argument("--mcep_alpha", default=0.41, type=float, help="Alpha of mel cepstrum")
    parser.add_argument("--highpass_cutoff", default=70, type=int, help="Cut off frequency in lowpass filter")
    parser.add_argument("--dtw", action="store_true", help="align each pair by dynamic time warping")
    parser.add_argument("--max_frame_diff", default=2, type=int,
                        help="largest frame-count difference of a pair compared without --dtw")
    parser.add_argument("--batch_size", default=64, type=int, help="pairs per kernel launch")
    parser.add_argument("--outfile", required=True, type=str, help="TSV file to write")
    parser.add_argument("--verbose", default=1, type=int, help="log level")
    return parser


def wav_list(arg):
    """The wav files of a directory (sorted) or of a list file."""
    if os.path.isdir(arg):
        return sorted(find_files(arg, "*.wav"))
    if os.path.isfile(arg):
        return read_txt(arg)
    raise ValueError("%s should be a directory or a list of wav files" % arg)


def wav_info(path):
    """(sampling rate, samples) of a wav file from its header."""
    from scipy.io import wavfile
    fs, x = wavfile.read(path, mmap=True)
    return int(fs), len(x)


def pair_files(ref_list, dec_list):
    """[(utterance id, reference wav, decoded wav)] paired by basename in the reference list's order, and the error
    messages for files without a counterpart or basenames given twice."""
    errors = []
    by_name = {}
    for side, files in (("reference", ref_list), ("decoded", dec_list)):
        seen = {}
        for f in files:
            b = os.path.basename(f)
            if b in seen:
                errors.append("%s wavs %s and %s have the same basename" % (side, seen[b], f))
            seen[b] = f
        by_name[side] = seen
    refs, decs = by_name["reference"], by_name["decoded"]
    for b, f in refs.items():
        if b not in decs:
            errors.append("reference wav %s has no decoded counterpart named %s" % (f, b))
    for b, f in decs.items():
        if b not in refs:
            errors.append("decoded wav %s has no reference counterpart named %s" % (f, b))
    pairs = [(os.path.splitext(b)[0], f, decs[b]) for b, f in refs.items() if b in decs]
    return pairs, errors


def check_pairs(pairs, info, fs, fftl, hop, max_frame_diff, dtw):
    """Error messages for every pair that cannot be compared: a sampling rate other than ``fs``, a wav shorter than
    ``fftl`` and, without ``dtw``, frame counts more than ``max_frame_diff`` apart.  ``info(path)`` gives (rate,
    samples)."""
    errors = []
    for _, ref, dec in pairs:
        (rfs, rn), (dfs, dn) = info(ref), info(dec)
        bad = False
        for f, r, n in ((ref, rfs, rn), (dec, dfs, dn)):
            if r != fs:
                errors.append("%s is sampled at %d Hz, not --fs %d" % (f, r, fs))
                bad = True
            if n < fftl:
                errors.append("%s has %d samples, fewer than --fftl %d, so it has no frames" % (f, n, fftl))
                bad = True
        if bad or dtw:
            continue
        tr, td = n_frames(rn, fftl, hop), n_frames(dn, fftl, hop)
        if abs(tr - td) > max_frame_diff:
            errors.append("%s has %d frames and %s has %d: more than --max_frame_diff %d apart; compare them along a "
                          "time-warping path with --dtw" % (ref, tr, dec, td, max_frame_diff))
    return errors


def _read(path):
    fs, x = read_wav_int16(path)
    return x


def compute(pairs, args):
    """``Mcd`` of every pair, ``--batch_size`` pairs per launch."""
    from pytorchwavenetvocoder_b200.utils.distortion import Mcd, mcd_wavs
    hop = shift_length(args.shiftms, args.fs)
    parts = []
    bs = max(int(args.batch_size), 1)
    for i0 in range(0, len(pairs), bs):
        batch = pairs[i0:i0 + bs]
        logging.info("pairs %d-%d of %d" % (i0 + 1, i0 + len(batch), len(pairs)))
        refs, decs = [_read(r) for _, r, _ in batch], [_read(d) for _, _, d in batch]
        for side in (refs, decs):
            if not all(x.dtype == np.int16 for x in side):
                side[:] = [np.asarray(x, dtype=np.float64) for x in side]
        parts.append(mcd_wavs(refs, decs, args.fs, args.fftl, hop, args.mcep_dim, args.mcep_alpha,
                              highpass_cutoff=args.highpass_cutoff, dtw=args.dtw))
    return Mcd(*(np.concatenate([getattr(p, f) for p in parts]) for f in ("mcd", "counts", "sums")), None)


def write_tsv(path, ids, result):
    """One row per utterance and a ``<corpus>`` row; values with 17 significant digits.  Returns corpus_mcd."""
    from pytorchwavenetvocoder_b200.utils.distortion import corpus_mcd
    corpus = corpus_mcd(result)
    with open(path, "w") as f:
        f.write("utt_id\tframes\tmcd_db\n")
        for u, n, m in zip(ids, result.counts, result.mcd):
            f.write("%s\t%d\t%.17g\n" % (u, n, m))
        f.write("<corpus>\t%d\t%.17g\n" % (int(np.sum(result.counts)), corpus[0]))
    return corpus


def main(argv=None):
    args = get_parser().parse_args(argv)
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    level = logging.INFO if args.verbose > 0 else logging.WARNING
    logging.basicConfig(level=logging.DEBUG if args.verbose > 1 else level, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    try:
        refs, decs = wav_list(args.reference), wav_list(args.decoded)
    except ValueError as e:
        logging.error(str(e))
        sys.exit(1)
    pairs, errors = pair_files(refs, decs)
    if not errors:
        errors = check_pairs(pairs, wav_info, args.fs, args.fftl, shift_length(args.shiftms, args.fs),
                             args.max_frame_diff, args.dtw)
    if not errors and not pairs:
        errors = ["no wav files to compare"]
    if errors:
        for e in errors:
            logging.error(e)
        logging.error("nothing was computed")
        sys.exit(1)
    import torch
    if not torch.cuda.is_available():
        logging.error("gpu is not available. please check the setting.")
        sys.exit(1)
    logging.info("comparing %d pairs %s" % (len(pairs), "along DTW paths" if args.dtw else "frame by frame"))
    result = compute(pairs, args)
    corpus, mean = write_tsv(args.outfile, [u for u, _, _ in pairs], result)
    logging.info("corpus MCD %.4f dB over %d %s (mean of %d utterances %.4f dB)"
                 % (corpus, int(np.sum(result.counts)), "path steps" if args.dtw else "frames", len(pairs), mean))


if __name__ == "__main__":
    main()
