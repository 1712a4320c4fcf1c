#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""RESYNTHESIZE WAVS THROUGH THE VOCODER -- analysis-synthesis with no feature files.

Each wav is read in chunks of ``--chunk_samples`` and pushed through ``MelspcStream`` (the low-cut filter and the log
mel-spectrogram of ``feature_extract.py --feature_type melspc``, scaled by the model's ``--stats``), whose frames feed a
decode session as they arrive; with ``--noise_shaping`` the PCM_16 samples go through the MLSA restoration filter; each
wav is written as its samples arrive.  The output bytes equal ``feature_extract.py --feature_type melspc --save_wav
false`` with the same analysis flags followed by ``decode.py`` with the same checkpoint, stats, batch size, seed,
``--decode_math`` and ``--noise_shaping``: the same length-sorted batches (from the wav headers), the same seed draws,
``n_samples = frames * upsampling_factor - 1``, and zero aux columns past a shorter row's end.  Within a batch the rows
of a session advance together, so each row's frames are buffered and the session is fed the frames every row has
(an ended row counts as having zeros up to the longest row).

The model must take these features as they come: ``feature_type`` melspc, an up-sampling layer with
``upsampling_factor`` equal to the frame shift, no speaker code, ``n_aux`` equal to the stats' mel count, and every wav
at ``--fs``.  Anything else exits 1 naming the mismatch, before anything is written."""
import argparse
import logging
import math
import os
import sys

import numpy as np
import torch

from pytorchwavenetvocoder_b200.bin.decode import SessionWriter, _restoration_filter, load_model, load_scaler
from pytorchwavenetvocoder_b200.bin.feature_extract import _optional_int
from pytorchwavenetvocoder_b200.nets import encode_mu_law
from pytorchwavenetvocoder_b200.utils import find_files, have_soundfile, read_hdf5, read_txt, read_wav_int16
from pytorchwavenetvocoder_b200.utils.melspc import MelspcStream, n_frames, shift_length


def get_parser():
    """decode.py's flags (without --feats, --n_gpus, --intervals, --chunk_frames), feature_extract.py's analysis flags
    with their defaults, and --chunk_samples."""
    parser = argparse.ArgumentParser(description="resynthesize wavs through a melspc WaveNet vocoder")
    parser.add_argument("--waveforms", required=True, type=str, help="directory or list of input wav files")
    parser.add_argument("--checkpoint", required=True, type=str, help="model file")
    parser.add_argument("--outdir", required=True, type=str, help="directory to save generated samples")
    parser.add_argument("--stats", default=None, type=str, help="hdf5 file including statistics")
    parser.add_argument("--config", default=None, type=str, help="configure file")
    parser.add_argument("--fs", default=16000, type=int, help="sampling rate")
    parser.add_argument("--batch_size", default=32, type=int, help="number of batch size in decoding")
    parser.add_argument("--seed", default=1, type=int, help="seed number")
    parser.add_argument("--verbose", default=1, type=int, help="log level")
    parser.add_argument("--decode_math", default="fp32", choices=["fp32", "bf16"],
                        help="decode precision: fp32 (default) or the bf16 tensor-core decoder of the 512/256-size models")
    parser.add_argument("--noise_shaping", action="store_true",
                        help="restore noise-shaped output with the MLSA filter of --stats (/mlsa/coef, /mlsa/alpha)")
    parser.add_argument("--shiftms", default=5, type=float, help="Frame shift in msec")
    parser.add_argument("--fftl", default=1024, type=int, help="FFT length")
    parser.add_argument("--fmin", default=None, nargs="?", type=_optional_int,
                        help="minimum frequency for melspc (empty: not given)")
    parser.add_argument("--fmax", default=None, nargs="?", type=_optional_int,
                        help="maximum frequency for melspc (empty: not given)")
    parser.add_argument("--highpass_cutoff", default=70, type=int, help="Cut off frequency in lowpass filter")
    parser.add_argument("--chunk_samples", default=0, type=int,
                        help="PCM samples pushed per call (0: the whole file); the files are the same either way")
    return parser


def _wav_header(path):
    """(sampling rate, sample count) of a wav file without reading its samples."""
    try:
        from scipy.io import wavfile
        fs, x = wavfile.read(path, mmap=True)
        return int(fs), len(x)
    except ImportError:
        import wave
        with wave.open(path, "rb") as w:
            return w.getframerate(), w.getnframes()


def check_setup(config, stats_mean_shape, hop, fs, wav_headers):
    """Every reason these wavs cannot go through this model as features, as messages (empty when there is none)."""
    errs = []
    if config.feature_type != "melspc":
        errs.append("the model takes feature_type %r features; resynthesis extracts melspc" % config.feature_type)
    if not config.use_upsampling_layer:
        errs.append("the model has no up-sampling layer; resynthesis feeds frame-rate aux features")
    elif hop != config.upsampling_factor:
        errs.append("frame shift %d samples (--shiftms at --fs) != the model's upsampling_factor %d"
                    % (hop, config.upsampling_factor))
    if config.use_speaker_code:
        errs.append("the model uses a speaker code; resynthesis has none")
    n_mels = stats_mean_shape[0] if len(stats_mean_shape) == 1 else None
    if n_mels != config.n_aux:
        errs.append("the stats hold %s mel bands but the model's n_aux is %d" % (n_mels, config.n_aux))
    for path, (wfs, _) in wav_headers:
        if wfs != fs:
            errs.append("%s is sampled at %d Hz, not --fs %d" % (path, wfs, fs))
    return errs


def batches(wav_list, frames, batch_size):
    """decode.py's batch order: the file order for batch size 1, else ``np.argsort`` of the frame counts split by
    ``np.array_split`` into ceil(n / batch_size) batches."""
    if batch_size == 1:
        return [[w] for w in wav_list]
    order = [wav_list[i] for i in np.argsort(frames)]
    return [f.tolist() for f in np.array_split(order, math.ceil(len(order) / batch_size))]


def resynthesize_batch(model, paths, outdir, args, config, scaler, shaping, pcm16):
    """One decode session over the wavs ``paths``: chunks -> MelspcStream -> session -> wav files."""
    hop = shift_length(args.shiftms, args.fs)
    U, n_mels, B = config.upsampling_factor, config.n_aux, len(paths)
    dev = torch.device("cuda", torch.cuda.current_device())
    wavs = [read_wav_int16(p)[1] for p in paths]
    if not all(w.dtype == np.int16 for w in wavs):
        wavs = [np.asarray(w, dtype=np.float64) for w in wavs]
    wavs = [torch.from_numpy(np.ascontiguousarray(w)).to(dev) for w in wavs]
    totals = [n_frames(w.numel(), hop) for w in wavs]
    seed = encode_mu_law(np.zeros(1), config.n_quantize)
    x = torch.from_numpy(np.stack([seed] * B, axis=0)).long().to(dev)
    ids = [os.path.basename(p).replace(".wav", "") for p in paths]
    stream = MelspcStream(args.fs, args.fftl, hop, n_mels, fmin=args.fmin, fmax=args.fmax,
                          highpass_cutoff=args.highpass_cutoff, scaler=(scaler.mean_, scaler.scale_), device=dev)
    sw = SessionWriter(model, x, [t * U - 1 for t in totals], [outdir + "/" + i + ".wav" for i in ids], args.fs,
                       config.n_quantize, pcm16, shaping)
    T = max(totals)
    bufs = [[] for _ in range(B)]     # each row's frames not yet fed
    got = [0] * B                     # frames received per row
    fed = 0
    pos = [0] * B
    step = args.chunk_samples if args.chunk_samples > 0 else max(w.numel() for w in wavs)
    try:
        while fed < T and not sw.sess.done:
            live = [b for b in range(B) if got[b] < totals[b]]
            if live:
                chunks = {b: wavs[b][pos[b]:pos[b] + step] for b in live}
                final = [b for b in live if pos[b] + step >= wavs[b].numel()]
                for b, a in stream.push(chunks, final).items():
                    bufs[b].append(a)
                    got[b] += a.size(1)
                    pos[b] += chunks[b].numel()
            # an ended row has every frame; past its end the session reads zeros, as pad_list gives them
            k = min(T if got[b] == totals[b] else got[b] for b in range(B)) - fed
            if k <= 0:
                continue
            h = torch.zeros(B, n_mels, k, dtype=torch.float32, device=dev)
            for b in range(B):
                have = torch.cat(bufs[b], 1) if len(bufs[b]) > 1 else (bufs[b][0] if bufs[b] else None)
                n = min(k, 0 if have is None else have.size(1))
                if n > 0:
                    h[b, :, :n] = have[:, :n]
                    bufs[b] = [have[:, n:]]
            sw.feed(h)
            fed += k
    finally:
        sw.close()
    return ids


def main(argv=None):
    """RUN RESYNTHESIS."""
    args = get_parser().parse_args(argv)
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    level = logging.INFO if args.verbose > 0 else logging.WARNING
    if args.verbose > 1:
        level = logging.DEBUG
    logging.basicConfig(level=level, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    for key, value in vars(args).items():
        logging.info("%s = %s" % (key, str(value)))
    if args.stats is None:
        args.stats = os.path.dirname(args.checkpoint) + "/stats.h5"
    if args.config is None:
        args.config = os.path.dirname(args.checkpoint) + "/model.conf"
    config = torch.load(args.config, weights_only=False)
    if os.path.isdir(args.waveforms):
        wav_list = sorted(find_files(args.waveforms, "*.wav"))
    elif os.path.isfile(args.waveforms):
        wav_list = read_txt(args.waveforms)
    else:
        logging.error("--waveforms should be directory or list.")
        sys.exit(1)
    hop = shift_length(args.shiftms, args.fs)
    headers = [(p, _wav_header(p)) for p in wav_list]
    mean_shape = np.shape(read_hdf5(args.stats, "/melspc/mean")) if config.feature_type == "melspc" else ()
    errs = check_setup(config, mean_shape, hop, args.fs, headers)
    if errs:
        for e in errs:
            logging.error(e)
        sys.exit(1)
    if not torch.cuda.is_available():
        logging.error("gpu is not available. please check the setting.")
        sys.exit(1)
    if not os.path.exists(args.outdir):
        os.makedirs(args.outdir)
    # decode.py's seeds (its one-GPU worker seeds again with seed + 0 before it draws anything)
    os.environ['PYTHONHASHSEED'] = str(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    shaping = _restoration_filter(args.stats) if args.noise_shaping else None
    pcm16 = args.batch_size > 1 and not have_soundfile()
    with torch.cuda.device(0):
        with torch.no_grad():
            model = load_model(args, config)
            scaler = load_scaler(args.stats, "melspc")
            for paths in batches(wav_list, [n_frames(n, hop) for _, (_, n) in headers], args.batch_size):
                ids = resynthesize_batch(model, paths, args.outdir, args, config, scaler, shaping, pcm16)
                logging.info("wrote %s in %s." % (", ".join(i + ".wav" for i in ids), args.outdir))


if __name__ == "__main__":
    main()
