#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""Noise shaping CLI (drop-in for reference wavenet_vocoder/bin/noise_shaping.py: same flags, same stats keys
``/mlsa/coef`` + ``/mlsa/alpha``, same int16 wav output) with the MLSA filter on the GPU: the wav list is processed in
batches of ``--batch_size`` files per kernel launch instead of ``--n_jobs`` CPU processes (``--n_jobs`` is accepted and
ignored).  Differences from the reference, both stated in DESIGN.md: every file starts from a zero filter state (the
reference's per-process filter object carries its state from one file into the next), and pysptk is not needed."""
import argparse
import logging
import os
import sys

import numpy as np

from pytorchwavenetvocoder_b200.utils import (check_hdf5, find_files, read_hdf5, read_txt, read_wav_int16, write_hdf5,
                                             write_wav_int16)
from pytorchwavenetvocoder_b200.utils.mlsa import convert_mcep_to_mlsa_coef, mlsa_filter_batch


def _strtobool(v):
    v = str(v).lower()
    if v in ("y", "yes", "t", "true", "on", "1"):
        return 1
    if v in ("n", "no", "f", "false", "off", "0"):
        return 0
    raise ValueError("invalid truth value %r" % (v,))


def noise_shaping(wav_list, args):
    """APPLY NOISE SHAPING BASED ON MLSA FILTER (reference noise_shaping.py:46-87), a batch of files per launch."""
    if check_hdf5(args.stats, "/mlsa/coef"):
        mlsa_coef = np.array(read_hdf5(args.stats, "/mlsa/coef"), dtype=np.float64)
        alpha = float(read_hdf5(args.stats, "/mlsa/alpha"))
    else:
        raise KeyError("\"/mlsa/coef\" is not found in %s." % (args.stats))
    if args.inv:
        mlsa_coef *= -1.0
    bs = max(int(getattr(args, "batch_size", 64)), 1)
    for i0 in range(0, len(wav_list), bs):
        names = wav_list[i0:i0 + bs]
        xs = []
        for i, wav_name in enumerate(names):
            logging.info("now processing %s (%d/%d)" % (wav_name, i0 + i + 1, len(wav_list)))
            fs, x = read_wav_int16(wav_name)
            if x.dtype != np.int16:
                logging.warning("wav file format is not 16 bit PCM.")
            if not fs == args.fs:
                logging.error("sampling frequency is not matched.")
                sys.exit(1)
            xs.append(x if x.dtype == np.int16 else np.float64(x))
        if not all(x.dtype == np.int16 for x in xs):
            xs = [np.float64(x) for x in xs]
        ys = mlsa_filter_batch(xs, mlsa_coef, alpha, pd=4, out_int16=True)
        for wav_name, y in zip(names, ys):
            write_wav_int16(args.outdir + "/" + os.path.basename(wav_name), args.fs, y)


def main(argv=None):
    """RUN NOISE SHAPING (reference noise_shaping.py:90-191)."""
    parser = argparse.ArgumentParser(description="making feature file argsurations.")
    parser.add_argument("--waveforms", default=None, help="directory or list of filename of input wavfile")
    parser.add_argument("--stats", default=None, help="filename of hdf5 format")
    parser.add_argument("--outdir", default=None, help="directory to save preprocessed wav file")
    parser.add_argument("--fs", default=16000, type=int, help="Sampling frequency")
    parser.add_argument("--shiftms", default=5, type=float, help="Frame shift in msec")
    parser.add_argument("--feature_type", default="world", choices=["world", "mcep", "melspc"], type=str, help="feature type")
    parser.add_argument("--mcep_dim_start", default=2, type=int, help="Start index of mel cepstrum")
    parser.add_argument("--mcep_dim_end", default=27, type=int, help="End index of mel cepstrum")
    parser.add_argument("--mcep_alpha", default=0.41, type=float, help="Alpha of mel cepstrum")
    parser.add_argument("--mag", default=0.5, type=float, help="magnification of noise shaping")
    parser.add_argument("--verbose", default=1, type=int, help="log message level")
    parser.add_argument("--n_jobs", default=10, type=int, help="number of parallel jobs (accepted, unused: one GPU launch per batch)")
    parser.add_argument("--batch_size", default=64, type=int, help="wav files per kernel launch")
    parser.add_argument("--inv", default=False, type=_strtobool, help="if True, inverse filtering will be performed")
    args = parser.parse_args(argv)

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

    if os.path.isdir(args.waveforms):
        file_list = sorted(find_files(args.waveforms, "*.wav"))
    else:
        file_list = read_txt(args.waveforms)
    logging.info("number of utterances = %d" % len(file_list))
    if not os.path.exists(args.outdir):
        os.makedirs(args.outdir)

    # calculate MLSA coef and save it (reference :171-177)
    if not check_hdf5(args.stats, "/mlsa/coef"):
        avg_mcep = np.array(read_hdf5(args.stats, args.feature_type + "/mean"), dtype=np.float64)
        if args.feature_type == "world":
            avg_mcep = avg_mcep[args.mcep_dim_start:args.mcep_dim_end]
        mlsa_coef = convert_mcep_to_mlsa_coef(avg_mcep, args.mag, args.mcep_alpha)
        write_hdf5(args.stats, "/mlsa/coef", mlsa_coef)
        write_hdf5(args.stats, "/mlsa/alpha", args.mcep_alpha)

    if args.feature_type == "melspc":
        raise NotImplementedError("currently, support only world and mcep.")   # (as the reference, :181-183)
    noise_shaping(file_list, args)


if __name__ == "__main__":
    main()
