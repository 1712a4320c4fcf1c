#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""SCORE HELD-OUT UTTERANCES -- the teacher-forced negative log-likelihood of each (wav, feature) pair under one or
more checkpoints: the training loss of ``train.py`` computed on audio the model has not seen (``utils/scoring.py``,
DESIGN.md section 6 row e1).

Inputs follow ``train.py`` (``--waveforms`` / ``--feats``: directories or lists) and ``decode.py`` (``--checkpoint``,
``--stats`` and ``--config`` defaulting to the checkpoint's directory).  ``--outfile`` gets one TSV row per checkpoint
and utterance (checkpoint, utterance id, scored positions, summed NLL in nats, nats per sample) and one ``<corpus>``
row per checkpoint (the sums added in list order, and their mean); an utterance with nothing to score has count 0 and
0 nats per sample.  With several checkpoints the best is logged.

``--n_gpus N`` splits the list with ``np.array_split``, one process per GPU; the main process concatenates the
per-utterance sums in list order before adding them, so every figure is bit-identical to one GPU.
"""
from __future__ import division

import argparse
import logging
import os
import sys

import numpy as np
import torch
import torch.multiprocessing as mp

from pytorchwavenetvocoder_b200.utils import check_hdf5
from pytorchwavenetvocoder_b200.utils import find_files
from pytorchwavenetvocoder_b200.utils import read_txt


def get_parser():
    parser = argparse.ArgumentParser()
    parser.add_argument("--waveforms", required=True, type=str, help="directory or list of wav files")
    parser.add_argument("--feats", required=True, type=str, help="directory or list of aux feat files")
    parser.add_argument("--checkpoint", required=True, nargs="+", type=str, help="model file(s) to score")
    parser.add_argument("--stats", default=None, type=str, help="hdf5 file including statistics")
    parser.add_argument("--config", default=None, type=str, help="configure file")
    parser.add_argument("--outfile", required=True, type=str, help="TSV file to write")
    parser.add_argument("--batch_samples", default=1 << 19, type=int,
                        help="samples per scoring batch (rows x longest row); longer utterances are scored in windows")
    parser.add_argument("--start", default=None, type=int,
                        help="first scored position of each utterance (default: the receptive field, as in training)")
    parser.add_argument("--math_mode", default=None, choices=["tf32", "fp32", "bf16"],
                        help="forward precision (default: the --math_mode the model was trained with)")
    parser.add_argument("--n_gpus", default=1, type=int, help="number of gpus")
    parser.add_argument("--verbose", default=1, type=int, help="log level")
    return parser


def file_lists(waveforms, feats):
    """(wav_list, feat_list) as ``train.py`` reads them: a directory of wavs with same-named ``.h5`` features, or two
    list files.  Raises ValueError for a missing input or lists of different lengths."""
    if os.path.isdir(waveforms):
        names = sorted(find_files(waveforms, "*.wav", use_dir_name=False))
        wav_list = [waveforms + "/" + n for n in names]
        feat_list = [feats + "/" + n.replace(".wav", ".h5") for n in names]
    elif os.path.isfile(waveforms):
        if not os.path.isfile(feats):
            raise ValueError("--feats should be a list when --waveforms is one: %s" % feats)
        wav_list, feat_list = read_txt(waveforms), read_txt(feats)
    else:
        raise ValueError("--waveforms should be directory or list: %s" % waveforms)
    if len(wav_list) != len(feat_list):
        raise ValueError("%d waveforms but %d feature files" % (len(wav_list), len(feat_list)))
    return wav_list, feat_list


def check_stats(stats, feature_type):
    """An error message when ``stats`` lacks the scaler of ``feature_type``, else None."""
    for key in ("/" + feature_type + "/mean", "/" + feature_type + "/scale"):
        if not check_hdf5(stats, key):
            return "%s has no %s: the model was trained on --feature_type %s" % (stats, key, feature_type)
    return None


def build_model(config, checkpoint, math_mode):
    """The WaveNet of ``checkpoint`` under ``config`` on the current device, with ``math_mode`` (``train.py``'s rule:
    tf32 falls back to fp32 for a shape the tensor-core path does not cover; bf16 is refused there)."""
    from pytorchwavenetvocoder_b200.bin.decode import load_model
    from pytorchwavenetvocoder_b200.nets.wavenet import bf16_supported, tc_supported
    model = load_model(argparse.Namespace(checkpoint=checkpoint), config)
    U = config.upsampling_factor if config.use_upsampling_layer else 0
    cfg_t = (config.n_quantize, config.n_aux, config.n_resch, config.n_skipch, config.dilation_depth,
             config.dilation_repeat, config.kernel_size, U)
    if math_mode == "bf16" and not bf16_supported(cfg_t):
        raise ValueError("--math_mode bf16 does not cover this model; use tf32 or fp32")
    model.math_mode = math_mode if (math_mode != "tf32" or tc_supported(cfg_t)) else "fp32"
    return model


def score_files(wav_list, feat_list, gpu, args, config):
    """Scores of one GPU's share: ``[(nll (N,), count (N,))]``, one pair per checkpoint, in list order."""
    from pytorchwavenetvocoder_b200.bin.decode import load_scaler
    from pytorchwavenetvocoder_b200.utils.scoring import load_utterance, score_utterances
    torch.cuda.set_device(gpu)
    if not wav_list:
        return [(np.zeros(0), np.zeros(0, dtype=np.int64)) for _ in args.checkpoint]
    scaler = load_scaler(args.stats, config.feature_type)
    utts = [load_utterance(w, f, config, scaler) for w, f in zip(wav_list, feat_list)]
    out = []
    for ckpt in args.checkpoint:
        model = build_model(config, ckpt, args.math_mode)
        out.append(score_utterances(model, utts, args.batch_samples, args.start))
        del model
    return out


def write_tsv(path, checkpoints, ids, scores):
    """One row per (checkpoint, utterance) and one ``<corpus>`` row per checkpoint.  An utterance with nothing to score
    (shorter than the first scored position) has count 0, NLL 0 and 0 nats per sample.  NLL sums are written with 17
    significant digits, so they read back as the float64 the scoring returned.  Returns the corpus means."""
    from pytorchwavenetvocoder_b200.utils.scoring import corpus_mean
    means = []
    with open(path, "w") as f:
        f.write("checkpoint\tutt_id\tcount\tnll_sum\tnats_per_sample\n")
        for ckpt, (nll, count) in zip(checkpoints, scores):
            for u, v, c in zip(ids, nll, count):
                f.write("%s\t%s\t%d\t%.17g\t%.17g\n" % (ckpt, u, c, v, v / c if c > 0 else 0.0))
            s, n, mean = corpus_mean(nll, count)
            f.write("%s\t<corpus>\t%d\t%.17g\t%.17g\n" % (ckpt, n, s, mean))
            means.append(mean)
    return means


def main(argv=None):
    args = get_parser().parse_args(argv)
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    level = logging.INFO if args.verbose > 0 else logging.WARNING
    logging.basicConfig(level=logging.DEBUG if args.verbose > 1 else level, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    if args.stats is None:
        args.stats = os.path.dirname(args.checkpoint[0]) + "/stats.h5"
    if args.config is None:
        args.config = os.path.dirname(args.checkpoint[0]) + "/model.conf"
    try:
        wav_list, feat_list = file_lists(args.waveforms, args.feats)
    except ValueError as e:
        logging.error(str(e))
        sys.exit(1)
    if args.batch_samples <= 0 or args.n_gpus <= 0:
        logging.error("--batch_samples and --n_gpus should be positive")
        sys.exit(1)
    config = torch.load(args.config, weights_only=False)
    if args.math_mode is None:
        args.math_mode = getattr(config, "math_mode", "tf32")
    refusal = check_stats(args.stats, config.feature_type)
    if refusal is not None:
        logging.error(refusal)
        sys.exit(1)
    if not torch.cuda.is_available():
        logging.error("gpu is not available. please check the setting.")
        sys.exit(1)
    logging.info("scoring %d utterances under %d checkpoint(s)" % (len(wav_list), len(args.checkpoint)))

    parts = np.array_split(np.arange(len(wav_list)), args.n_gpus)
    shares = [([wav_list[i] for i in p], [feat_list[i] for i in p]) for p in parts]
    if args.n_gpus == 1:
        results = [score_files(shares[0][0], shares[0][1], 0, args, config)]
    else:
        with mp.get_context("spawn").Pool(args.n_gpus) as pool:
            results = pool.starmap(score_files, [(w, f, g, args, config) for g, (w, f) in enumerate(shares)])
    scores = [(np.concatenate([r[c][0] for r in results]), np.concatenate([r[c][1] for r in results]))
              for c in range(len(args.checkpoint))]
    ids = [os.path.basename(f).replace(".h5", "").replace(".npz", "") for f in feat_list]
    means = write_tsv(args.outfile, args.checkpoint, ids, scores)
    for ckpt, mean in zip(args.checkpoint, means):
        logging.info("%s: %.6f nats / sample" % (ckpt, mean))
    if len(args.checkpoint) > 1:
        best = min(range(len(means)), key=lambda c: (np.isnan(means[c]), means[c]))
        logging.info("best checkpoint: %s (%.6f nats / sample)" % (args.checkpoint[best], means[best]))


if __name__ == "__main__":
    main()
