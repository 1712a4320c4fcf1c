#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""DECODE WITH WAVENET VOCODER -- H100 build of ``wavenet_vocoder/bin/decode.py`` (reference v0.1.1).

Same flags (reference decode.py:179-204), same inputs (``model.conf``, ``checkpoint*.pkl`` with key
``"model"``, feature ``.h5`` files, ``stats.h5``) and outputs (``{feat_id}.wav`` PCM_16 at ``--fs``).
Utterances are length-sorted and batched like the reference (``decode_generator`` :52-174) and sharded over
GPUs with ``np.array_split`` (:261-262), one process per GPU, no communication (:330-338).  Each batch
is ONE persistent-kernel launch (``WaveNet.batch_fast_generate``); like the reference the decoding mode is
"sampling".

With ``--pool_capacity C`` each GPU worker instead decodes its whole file list through one continuous-batching pool
of C rows (``WaveNet.decode_pool(C, "sampling")``, under either ``--decode_math``; under fp32 a model the warp decoder
does not cover runs on the streaming decoder, ``kernel="stream"``): files enter free rows longest
first as others finish, so no row idles until the longest file of a batch ends.  The stream id of a file is its index
in the worker's list and the pool seed is ``pool_seed(--seed, gpu)``; each ``{feat_id}.wav`` holds exactly the samples
the pool API gives for the same model, seed and features (``decode_pool_files``).
"""
from __future__ import division

import argparse
import logging
import math
import os
import sys

import numpy as np
import torch
import torch.multiprocessing as mp

from sklearn.preprocessing import StandardScaler

from pytorchwavenetvocoder_b200.nets import decode_mu_law
from pytorchwavenetvocoder_b200.nets import encode_mu_law
from pytorchwavenetvocoder_b200.nets import WaveNet
from pytorchwavenetvocoder_b200.nets.wavenet import warp_pool_supported
from pytorchwavenetvocoder_b200.utils import extend_time
from pytorchwavenetvocoder_b200.utils import find_files
from pytorchwavenetvocoder_b200.utils import read_hdf5
from pytorchwavenetvocoder_b200.utils import read_txt
from pytorchwavenetvocoder_b200.utils import shape_hdf5
from pytorchwavenetvocoder_b200.utils import have_soundfile
from pytorchwavenetvocoder_b200.utils import write_wav
from pytorchwavenetvocoder_b200.utils import write_wav_pcm16
from pytorchwavenetvocoder_b200.utils import WavWriter
from pytorchwavenetvocoder_b200.utils import check_hdf5
from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter


def pad_list(batch_list, pad_value=0.0):
    """PAD VALUE (reference decode.py:31-49): list of (T_i, C) -> (B, T_max, C), zero padded like there."""
    maxlen = max(b.shape[0] for b in batch_list)
    out = np.zeros((len(batch_list), maxlen, batch_list[0].shape[-1]))
    for i, b in enumerate(batch_list):
        out[i, :b.shape[0]] = b
    return out


def _load_feat(featfile, feature_type, upsampling_factor, use_upsampling_layer, use_speaker_code, feat_transform):
    h = read_hdf5(featfile, "/" + feature_type)
    if not use_upsampling_layer:
        h = extend_time(h, upsampling_factor)
    if use_speaker_code:
        sc = read_hdf5(featfile, "/speaker_code")
        h = np.concatenate([h, np.tile(sc, [h.shape[0], 1])], axis=1)
    if feat_transform is not None:
        h = feat_transform(h)
    n_samples = h.shape[0] - 1 if not use_upsampling_layer else h.shape[0] * upsampling_factor - 1
    return h, n_samples


def decode_generator(feat_list,
                     batch_size=32,
                     feature_type="world",
                     wav_transform=None,
                     feat_transform=None,
                     upsampling_factor=80,
                     use_upsampling_layer=True,
                     use_speaker_code=False):
    """GENERATE DECODING BATCH (reference decode.py:52-174).

    batch_size == 1: yields ``feat_id, (x (1,1), h (1,C,T), n_samples)`` per file;
    otherwise length-sorted batches ``feat_ids, (x (B,1), h (B,C,T_max), n_samples_list)``.
    The seed sample is ``wav_transform(0)`` (= 128 for mu-law 256)."""
    def seed():
        x = np.zeros((1))
        return wav_transform(x) if wav_transform is not None else x

    def cuda(t):
        return t.cuda() if torch.cuda.is_available() else t

    if batch_size == 1:
        for featfile in feat_list:
            h, n_samples = _load_feat(featfile, feature_type, upsampling_factor, use_upsampling_layer,
                                      use_speaker_code, feat_transform)
            x = torch.from_numpy(np.asarray(seed())).long().unsqueeze(0)
            ht = torch.from_numpy(np.asarray(h)).float().transpose(0, 1).unsqueeze(0)
            feat_id = os.path.basename(featfile).replace(".h5", "").replace(".npz", "")
            yield feat_id, (cuda(x), cuda(ht), n_samples)
    else:
        shape_list = [shape_hdf5(f, "/" + feature_type)[0] for f in feat_list]
        feat_list = [feat_list[i] for i in np.argsort(shape_list)]
        n_batch = math.ceil(len(feat_list) / batch_size)
        for batch_list in [f.tolist() for f in np.array_split(feat_list, n_batch)]:
            batch_x, batch_h, n_samples_list, feat_ids = [], [], [], []
            for featfile in batch_list:
                h, n_samples = _load_feat(featfile, feature_type, upsampling_factor, use_upsampling_layer,
                                          use_speaker_code, feat_transform)
                batch_x.append(seed())
                batch_h.append(h)
                n_samples_list.append(n_samples)
                feat_ids.append(os.path.basename(featfile).replace(".h5", "").replace(".npz", ""))
            bx = torch.from_numpy(np.stack(batch_x, axis=0)).long()
            bh = torch.from_numpy(pad_list(batch_h)).float().transpose(1, 2)
            yield feat_ids, (cuda(bx), cuda(bh), n_samples_list)


def get_parser():
    """Flags of reference decode.py:179-204."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--feats", required=True, type=str, help="list or directory of aux feat files")
    parser.add_argument("--checkpoint", required=True, type=str, help="model file")
    parser.add_argument("--outdir", required=True, type=str, help="directory to save generated samples")
    parser.add_argument("--stats", default=None, type=str, help="hdf5 file including statistics")
    parser.add_argument("--config", default=None, type=str, help="configure file")
    parser.add_argument("--fs", default=16000, type=int, help="sampling rate")
    parser.add_argument("--batch_size", default=32, type=int, help="number of batch size in decoding")
    parser.add_argument("--n_gpus", default=1, type=int, help="number of gpus")
    parser.add_argument("--intervals", default=1000, type=int, help="log interval")
    parser.add_argument("--seed", default=1, type=int, help="seed number")
    parser.add_argument("--verbose", default=1, type=int, help="log level")
    parser.add_argument("--decode_math", default="fp32", choices=["fp32", "bf16"],
                        help="decode precision: fp32 (default) or the bf16 tensor-core decoder of the 512/256-size models")
    parser.add_argument("--chunk_frames", default=0, type=int,
                        help="decode through a resumable session, feeding this many aux frames per call and writing each "
                             "wav as its samples arrive (0: one launch per batch); the files are the same either way")
    parser.add_argument("--noise_shaping", action="store_true",
                        help="restore noise-shaped output with the MLSA filter of --stats (/mlsa/coef, /mlsa/alpha), as "
                             "noise_shaping.py --inv false does on the wav files; with --chunk_frames each chunk is "
                             "filtered as it arrives")
    parser.add_argument("--pool_capacity", default=0, type=int,
                        help="decode each GPU's files through one continuous-batching pool of this many rows, writing "
                             "each wav as its samples arrive (0: length-sorted batches of --batch_size)")
    return parser


def check_args(args):
    """Refusals of flag combinations, before anything is written: an error message, or None."""
    if args.pool_capacity < 0:
        return "--pool_capacity should be 0 (off) or a positive number of rows, got %d" % args.pool_capacity
    if args.pool_capacity > 0 and args.chunk_frames > 0:
        return ("--pool_capacity and --chunk_frames do not combine: the pool already writes each wav as its samples "
                "arrive, and every frame of a file is present when it is admitted")
    return None


def pool_seed(seed, gpu):
    """The decode-pool seed of GPU worker ``gpu`` for ``--seed``: the first 64-bit draw of torch's generator after
    ``torch.manual_seed(seed + gpu)``, the worker's own seeding."""
    torch.manual_seed(seed + gpu)
    return int(torch.empty((), dtype=torch.int64).random_().item())


def pool_kernel_for(model, capacity):
    """The decoder of ``--pool_capacity``: "stream" under fp32 when the warp decoder does not cover the model, else
    "auto" (the warp decoder under fp32, the bf16 decoder under bf16)."""
    if getattr(model, "decode_math", "fp32") == "fp32" and not warp_pool_supported(model, capacity):
        return "stream"
    return "auto"


def decode_pool_files(model, frames, capacity, seed, load, paths, fs, n_quantize, pcm16, shaping=None, kernel="auto"):
    """Decode files 0 .. len(frames) - 1 through one ``model.decode_pool(capacity, "sampling", seed, kernel=kernel)``
    and append each stream's samples to its wav (``paths[i]``) as calls return them; a writer closes when its stream
    finishes.

    ``load(i)`` -> (h (n_aux, frames) on the GPU, n_samples) reads file i; the stream id is i.  Files are admitted
    longest first (``frames[i]`` from the file shapes) and loaded lazily: at most 2 * capacity streams are admitted and
    unfinished at a time.  A stream's codes do not depend on when or into which row it is admitted, so the files are
    those of the pool API for the same seed and features.  ``pcm16`` or ``shaping``: PCM_16 from ``step_pcm16`` (and,
    with ``shaping`` = (coef, alpha), through one ``MlsaStreamFilter`` keyed by stream id); otherwise ``decode_mu_law``
    and the wav writer's quantisation."""
    order = iter(sorted(range(len(frames)), key=lambda i: (-frames[i], i)))
    pool = model.decode_pool(capacity, "sampling", seed, kernel=kernel)
    filt = MlsaStreamFilter(shaping[0], shaping[1], 4) if shaping is not None else None
    x = torch.full((1,), int(encode_mu_law(np.zeros(1), n_quantize)[0]), dtype=torch.int64, device="cuda")
    writers = {}
    try:
        while True:
            while len(writers) < 2 * capacity:
                i = next(order, None)
                if i is None:
                    break
                h, n_samples = load(i)
                writers[i] = WavWriter(paths[i], fs)
                pool.admit(x, n_samples, h, stream=i)
            if not writers:
                return
            out = (pool.step_pcm16 if pcm16 or filt is not None else pool.step)()
            if not out:   # every frame of an admitted file is present, so some stream can always run
                raise RuntimeError("decode pool: no stream could run")
            if filt is not None:
                out = filt.filter(out)
            for sid, y in out.items():
                y = y.cpu().numpy()
                if pcm16 or filt is not None:
                    writers[sid].write_pcm16(y)
                else:
                    writers[sid].write(decode_mu_law(y.astype(np.int64), n_quantize))
                if pool.finished(sid):
                    writers.pop(sid).close()
                    if filt is not None:
                        filt.close(sid)
                    logging.info("wrote %s." % paths[sid])
    finally:
        for w in writers.values():
            w.close()


def _restoration_filter(stats):
    """(coef, alpha) of the noise-shaping restoration (``noise_shaping.py --inv false``: +coef, pd 4)."""
    if not check_hdf5(stats, "/mlsa/coef"):
        raise KeyError("\"/mlsa/coef\" is not found in %s." % stats)
    return np.array(read_hdf5(stats, "/mlsa/coef"), dtype=np.float64), float(read_hdf5(stats, "/mlsa/alpha"))


class SessionWriter(object):
    """A ``WaveNet.decode_session`` over one batch whose new samples are appended to each utterance's wav as they
    arrive: ``feed(h_chunk)`` runs one session step and writes what it returned.

    ``shaping`` = (coef, alpha): pass each chunk's PCM_16 samples through the MLSA restoration filter on the device
    first (``MlsaStreamFilter``, rows as keys), which gives the samples ``noise_shaping.py --inv false`` gives for the
    whole file."""

    def __init__(self, model, x, n_samples_list, paths, fs, n_quantize, pcm16, shaping=None):
        self.sess = model.decode_session(x, n_samples_list, "sampling")
        self.filt = MlsaStreamFilter(shaping[0], shaping[1], 4, x.device) if shaping is not None else None
        self.writers = [WavWriter(p, fs) for p in paths]
        self.n_quantize, self.pcm16 = n_quantize, pcm16

    def feed(self, h_chunk):
        sess, filt = self.sess, self.filt
        out = (sess.step_pcm16 if self.pcm16 or filt is not None else sess.step)(h_chunk)
        counts = sess.last_counts
        if max(counts) == 0:
            return
        if filt is not None:
            ys = filt.filter({b: out[b, :c] for b, c in enumerate(counts) if c > 0})
            for b, y in ys.items():
                self.writers[b].write_pcm16(y.cpu().numpy())
            return
        out = out.cpu().numpy()
        for b, w in enumerate(self.writers):
            if counts[b] == 0:
                continue
            if self.pcm16:
                w.write_pcm16(out[b, :counts[b]])
            else:
                w.write(decode_mu_law(out[b, :counts[b]].astype(np.int64), self.n_quantize))

    def close(self):
        for w in self.writers:
            w.close()


def _decode_chunked(model, x, h, n_samples_list, chunk_frames, paths, fs, n_quantize, pcm16, shaping=None):
    """Decode one batch through ``WaveNet.decode_session`` in chunks of ``chunk_frames`` aux frames and append every
    utterance's new samples to its wav as they arrive (``SessionWriter``).  Same samples (hence same files) as the
    one-shot path."""
    sw = SessionWriter(model, x, n_samples_list, paths, fs, n_quantize, pcm16, shaping)
    try:
        for f0 in range(0, h.size(2), chunk_frames):
            if sw.sess.done:
                break
            sw.feed(h[:, :, f0:f0 + chunk_frames])
        if not sw.sess.done:   # the one-shot path raises the same way instead of writing short files
            raise ValueError("aux features too short: %d frames for %d samples" % (h.size(2), max(n_samples_list)))
    finally:
        sw.close()


def load_model(args, config):
    """The WaveNet of ``args.checkpoint`` built from ``config`` (model.conf), in eval mode on the current device, with
    ``args.decode_math``."""
    upsampling_factor = config.upsampling_factor if config.use_upsampling_layer else 0
    model = WaveNet(
        n_quantize=config.n_quantize,
        n_aux=config.n_aux,
        n_resch=config.n_resch,
        n_skipch=config.n_skipch,
        dilation_depth=config.dilation_depth,
        dilation_repeat=config.dilation_repeat,
        kernel_size=config.kernel_size,
        upsampling_factor=upsampling_factor)
    model.load_state_dict(torch.load(
        args.checkpoint, map_location=lambda storage, loc: storage, weights_only=False)["model"])
    model.eval()
    model.cuda()
    model.decode_math = getattr(args, "decode_math", "fp32")
    return model


def load_scaler(stats, feature_type):
    """The ``StandardScaler`` of ``stats`` (``/<feature_type>/mean`` and ``/scale``)."""
    scaler = StandardScaler()
    scaler.mean_ = read_hdf5(stats, "/" + feature_type + "/mean")
    scaler.scale_ = read_hdf5(stats, "/" + feature_type + "/scale")
    return scaler


def gpu_decode(feat_list, gpu, args, config):
    """One process per GPU (reference decode.py:274-327)."""
    # spawned workers do not inherit main()'s RNG state (the reference forks after seeding, decode.py:242):
    # re-seed here so that --seed controls the Philox stream of every GPU (distinct per GPU, reproducible)
    np.random.seed(args.seed + gpu)
    torch.manual_seed(args.seed + gpu)
    capacity = getattr(args, "pool_capacity", 0)
    seed = pool_seed(args.seed, gpu) if capacity > 0 else None
    with torch.cuda.device(gpu):
        with torch.no_grad():
            model = load_model(args, config)
            scaler = load_scaler(args.stats, config.feature_type)
            if capacity > 0:
                logging.info("decoding %d files through a pool of %d rows (seed %d); --batch_size is not used"
                             % (len(feat_list), capacity, seed))

                def load(i):
                    h, n = _load_feat(feat_list[i], config.feature_type, config.upsampling_factor,
                                      config.use_upsampling_layer, config.use_speaker_code, scaler.transform)
                    return torch.from_numpy(np.asarray(h)).float().t().contiguous().cuda(), n

                frames = [shape_hdf5(f, "/" + config.feature_type)[0] for f in feat_list]
                paths = [args.outdir + "/" + os.path.basename(f).replace(".h5", "").replace(".npz", "") + ".wav"
                         for f in feat_list]
                shaping = _restoration_filter(args.stats) if getattr(args, "noise_shaping", False) else None
                decode_pool_files(model, frames, capacity, seed, load, paths, args.fs, config.n_quantize,
                                  not have_soundfile(), shaping, pool_kernel_for(model, capacity))
                return
            generator = decode_generator(
                feat_list,
                batch_size=args.batch_size,
                feature_type=config.feature_type,
                wav_transform=lambda x: encode_mu_law(x, config.n_quantize),
                feat_transform=lambda x: scaler.transform(x),
                upsampling_factor=config.upsampling_factor,
                use_upsampling_layer=config.use_upsampling_layer,
                use_speaker_code=config.use_speaker_code)
            chunk = getattr(args, "chunk_frames", 0)
            # noise shaping filters the decoder's own PCM_16 samples (device quantisation, with or without soundfile);
            # without --chunk_frames the batch is decoded as one chunk holding every frame, i.e. one-shot decoding
            shaping = _restoration_filter(args.stats) if getattr(args, "noise_shaping", False) else None
            if args.batch_size > 1:
                for feat_ids, (batch_x, batch_h, n_samples_list) in generator:
                    logging.info("decoding start")
                    if chunk > 0 or shaping is not None:
                        _decode_chunked(model, batch_x, batch_h, n_samples_list, chunk or batch_h.size(2),
                                        [args.outdir + "/" + f + ".wav" for f in feat_ids], args.fs, config.n_quantize,
                                        not have_soundfile(), shaping)
                        logging.info("wrote %d wavs in %s." % (len(feat_ids), args.outdir))
                        continue
                    # batch_fast_generate returns completion order = ascending length, ties by batch index
                    order = sorted(range(len(feat_ids)), key=lambda b: (n_samples_list[b], b))
                    if not have_soundfile():
                        # the PCM_16 quantisation is ours (stdlib writer): do decode_mu_law + quantisation for the whole
                        # batch on the device and move 2 bytes per sample (reference :316-319 does both on the host)
                        pcm_list = model.batch_fast_generate_pcm16(batch_x, batch_h, n_samples_list, args.intervals)
                        for b, pcm in zip(order, pcm_list):
                            write_wav_pcm16(args.outdir + "/" + feat_ids[b] + ".wav", pcm, args.fs)
                            logging.info("wrote %s.wav in %s." % (feat_ids[b], args.outdir))
                        continue
                    samples_list = model.batch_fast_generate(batch_x, batch_h, n_samples_list, args.intervals)
                    for b, samples in zip(order, samples_list):
                        wav = decode_mu_law(samples, config.n_quantize)
                        write_wav(args.outdir + "/" + feat_ids[b] + ".wav", wav, args.fs)   # libsndfile quantises
                        logging.info("wrote %s.wav in %s." % (feat_ids[b], args.outdir))
            else:
                for feat_id, (x, h, n_samples) in generator:
                    logging.info("decoding %s (length = %d)" % (feat_id, n_samples))
                    if chunk > 0 or shaping is not None:
                        _decode_chunked(model, x, h, [n_samples], chunk or h.size(2),
                                        [args.outdir + "/" + feat_id + ".wav"], args.fs, config.n_quantize, False, shaping)
                        logging.info("wrote %s.wav in %s." % (feat_id, args.outdir))
                        continue
                    samples = model.fast_generate(x, h, n_samples, args.intervals)
                    wav = decode_mu_law(samples, config.n_quantize)
                    write_wav(args.outdir + "/" + feat_id + ".wav", wav, args.fs)
                    logging.info("wrote %s.wav in %s." % (feat_id, args.outdir))


def main():
    """RUN DECODING."""
    args = get_parser().parse_args()
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    level = logging.INFO if args.verbose > 0 else logging.WARNING
    if args.verbose > 1:
        level = logging.DEBUG
    logging.basicConfig(level=level, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    if args.verbose < 1:
        logging.warning("logging is disabled.")
    for key, value in vars(args).items():
        logging.info("%s = %s" % (key, str(value)))
    refusal = check_args(args)
    if refusal is not None:
        logging.error(refusal)
        sys.exit(1)
    if args.stats is None:
        args.stats = os.path.dirname(args.checkpoint) + "/stats.h5"      # reference decode.py:226-227
    if args.config is None:
        args.config = os.path.dirname(args.checkpoint) + "/model.conf"   # :228-229
    if not os.path.exists(args.outdir):
        os.makedirs(args.outdir)
    os.environ['PYTHONHASHSEED'] = str(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)

    config = torch.load(args.config, weights_only=False)   # argparse.Namespace written by train.py

    if os.path.isdir(args.feats):
        feat_list = sorted(find_files(args.feats, "*.h5")) or sorted(find_files(args.feats, "*.npz"))
    elif os.path.isfile(args.feats):
        feat_list = read_txt(args.feats)
    else:
        logging.error("--feats should be directory or list.")
        sys.exit(1)
    if not torch.cuda.is_available():
        logging.error("gpu is not available. please check the setting.")
        sys.exit(1)

    # utterance sharding: np.array_split over GPUs, one process each, no communication
    feat_lists = [f.tolist() for f in np.array_split(feat_list, args.n_gpus)]
    if args.n_gpus == 1:
        gpu_decode(feat_lists[0], 0, args, config)
        return
    ctx = mp.get_context("spawn")
    processes = []
    for gpu, f in enumerate(feat_lists):
        p = ctx.Process(target=gpu_decode, args=(f, gpu, args, config))
        p.start()
        processes.append(p)
    code = 0
    for p in processes:
        p.join()
        code = code or p.exitcode
    if code:
        logging.error("a decoding process failed (exit code %s)." % code)
        sys.exit(1)


if __name__ == "__main__":
    main()
