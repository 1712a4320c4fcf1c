#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""TRAIN WAVENET VOCODER -- H100 build of ``wavenet_vocoder/bin/train.py`` (reference v0.1.1).

Same command line (reference train.py:337-394), same ``model.conf`` / ``checkpoint-*.pkl`` formats
(:315-332, :429, :564-568), same batching arithmetic (``train_generator`` :67-312), same loop (:530-561).
What changes underneath: ``WaveNet`` is the sm_90a kernel build, the loss is the fused CE kernel, and
``--n_gpus N`` means N *processes* (the command re-launches itself under ``torch.distributed.run``; one rank per
GPU, a single flat NCCL all-reduce of the gradients per step) instead of single-process ``nn.DataParallel``
(:449-454).  ``--batch_size`` stays the GLOBAL batch: every rank trains on ``batch_size / n_gpus`` windows of it.  Extra, optional flags: ``--math_mode {tf32,fp32,bf16}``.
"""
from __future__ import division

import argparse
import logging
import os
import sys
import time

import numpy as np
import torch

from sklearn.preprocessing import StandardScaler

from pytorchwavenetvocoder_b200.nets import encode_mu_law
from pytorchwavenetvocoder_b200.nets import initialize
from pytorchwavenetvocoder_b200.nets import WaveNet
from pytorchwavenetvocoder_b200.utils import background
from pytorchwavenetvocoder_b200.utils import extend_time
from pytorchwavenetvocoder_b200.utils import find_files
from pytorchwavenetvocoder_b200.utils import read_hdf5
from pytorchwavenetvocoder_b200.utils import read_txt
from pytorchwavenetvocoder_b200.utils import read_wav


def validate_length(x, y, upsampling_factor=None):
    """VALIDATE LENGTH (reference train.py:35-64): trim waveform / features to matching lengths."""
    if upsampling_factor is None:
        n = min(x.shape[0], y.shape[0])
        x, y = x[:n], y[:n]
        assert len(x) == len(y)
    else:
        if x.shape[0] > y.shape[0] * upsampling_factor:
            x = x[:y.shape[0] * upsampling_factor]
        if x.shape[0] < y.shape[0] * upsampling_factor:
            mod_y = y.shape[0] * upsampling_factor - x.shape[0]
            mod_y_frame = mod_y // upsampling_factor + 1
            y = y[:-mod_y_frame]
            x = x[:y.shape[0] * upsampling_factor]
        assert len(x) == len(y) * upsampling_factor
    return x, y


def _load_pair(wavfile, featfile, feature_type, upsampling_factor, use_upsampling_layer, use_speaker_code):
    """One utterance: waveform float32 and aux features (frames, dims) (reference train.py:119-138)."""
    x, _ = read_wav(wavfile, dtype=np.float32)
    h = read_hdf5(featfile, "/" + feature_type)
    if not use_upsampling_layer:
        h = extend_time(h, upsampling_factor)
    if use_speaker_code:
        sc = read_hdf5(featfile, "/speaker_code")
        h = np.concatenate([h, np.tile(sc, [h.shape[0], 1])], axis=1)
    if use_upsampling_layer:
        return validate_length(x, h, upsampling_factor)
    return validate_length(x, h)


def _to_batch(xs, hs, ts):
    bx, bh, bt = torch.stack(xs), torch.stack(hs), torch.stack(ts)
    if torch.cuda.is_available():
        bx, bh, bt = bx.cuda(), bh.cuda(), bt.cuda()
    return (bx, bh), bt


@background(max_prefetch=16)
def train_generator(wav_list, feat_list, receptive_field,
                    batch_length=None,
                    batch_size=1,
                    feature_type="world",
                    wav_transform=None,
                    feat_transform=None,
                    shuffle=True,
                    upsampling_factor=80,
                    use_upsampling_layer=True,
                    use_speaker_code=False,
                    device=None):
    """GENERATE TRAINING BATCH (reference train.py:67-312; the four batching modes, same arithmetic).

    Yields ``((x, h), t)``: x (B, T) long inputs, h (B, D, T or T/upsampling_factor) float aux, t (B, T)
    next-sample targets.  Windows are ``receptive_field + batch_length`` long and hop by ``batch_length``.
    """
    if device is not None and torch.cuda.is_available():
        torch.cuda.set_device(device)   # this body runs in the prefetch thread: bind it to the rank's GPU
    if shuffle:
        idx = np.random.permutation(len(wav_list))
        wav_list = [wav_list[i] for i in idx]
        feat_list = [feat_list[i] for i in idx]
    if batch_length is not None and use_upsampling_layer:
        batch_mod = (receptive_field + batch_length) % upsampling_factor
        logging.warning("batch length is decreased due to upsampling (%d -> %d)" % (
            batch_length, batch_length - batch_mod))
        batch_length -= batch_mod
    if batch_length is None and batch_size > 1:
        logging.warning("in utterance batch mode, batchsize will be 1.")

    def prep(x_, h_):
        if wav_transform is not None:
            x_ = wav_transform(x_)
        if feat_transform is not None:
            h_ = feat_transform(h_)
        return torch.from_numpy(np.asarray(x_)).long(), torch.from_numpy(np.asarray(h_)).float()

    x_buffer = h_buffer = None
    while True:
        bx, bh, bt = [], [], []
        for wavfile, featfile in zip(wav_list, feat_list):
            x, h = _load_pair(wavfile, featfile, feature_type, upsampling_factor, use_upsampling_layer,
                              use_speaker_code)
            if batch_length is not None:
                # ---- mini-batch modes: slide a window over the concatenation of all utterances ----
                if x_buffer is None:
                    x_buffer = np.empty((0), dtype=np.float32)
                    h_buffer = np.empty((0, h.shape[1]), dtype=np.float32)
                x_buffer = np.concatenate([x_buffer, x], axis=0)
                h_buffer = np.concatenate([h_buffer, h], axis=0)
                if not use_upsampling_layer:
                    win = receptive_field + batch_length
                    while len(x_buffer) > win:
                        x_, h_ = prep(x_buffer[:win], h_buffer[:win])
                        bx.append(x_[:-1])
                        bh.append(h_[:-1].transpose(0, 1))
                        bt.append(x_[1:])
                        x_buffer, h_buffer = x_buffer[batch_length:], h_buffer[batch_length:]
                        if len(bx) == batch_size:
                            yield _to_batch(bx, bh, bt)
                            bx, bh, bt = [], [], []
                else:
                    h_bs = (receptive_field + batch_length) // upsampling_factor
                    x_bs = h_bs * upsampling_factor + 1
                    h_ss = batch_length // upsampling_factor
                    x_ss = h_ss * upsampling_factor
                    while len(h_buffer) > h_bs:
                        x_, h_ = prep(x_buffer[:x_bs], h_buffer[:h_bs])
                        bh.append(h_.transpose(0, 1))
                        bx.append(x_[:-1])
                        bt.append(x_[1:])
                        h_buffer, x_buffer = h_buffer[h_ss:], x_buffer[x_ss:]
                        if len(bx) == batch_size:
                            yield _to_batch(bx, bh, bt)
                            bx, bh, bt = [], [], []
            elif not use_upsampling_layer:
                # ---- utterance batch, aux already at sample rate ----
                x_, h_ = prep(x, h)
                yield _to_batch([x_[:-1]], [h_[:-1].transpose(0, 1)], [x_[1:]])
            else:
                # ---- utterance batch with the upsampling layer: drop the last frame ----
                x_, h_ = prep(x[:-upsampling_factor + 1], h[:-1])
                yield _to_batch([x_[:-1]], [h_.transpose(0, 1)], [x_[1:]])
        if shuffle:
            idx = np.random.permutation(len(wav_list))
            wav_list = [wav_list[i] for i in idx]
            feat_list = [feat_list[i] for i in idx]


def save_checkpoint(checkpoint_dir, model, optimizer, iterations):
    """SAVE CHECKPOINT (reference train.py:315-332): {"model", "optimizer", "iterations"}."""
    checkpoint = {
        "model": model.state_dict(),
        "optimizer": optimizer.state_dict(),
        "iterations": iterations}
    if not os.path.exists(checkpoint_dir):
        os.makedirs(checkpoint_dir)
    torch.save(checkpoint, checkpoint_dir + "/checkpoint-%d.pkl" % iterations)
    logging.info("%d-iter checkpoint created." % iterations)


def get_parser():
    """Flags of reference train.py:337-394 (+ optional --math_mode)."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--waveforms", required=True, type=str, help="directory or list of wav files")
    parser.add_argument("--feats", default=None, type=str,
                        help="directory or list of aux feat files (required unless --extract_features true)")
    parser.add_argument("--stats", default=None, type=str,
                        help="hdf5 file including statistics (required unless --extract_features true)")
    parser.add_argument("--expdir", required=True, type=str, help="directory to save the model")
    parser.add_argument("--feature_type", default="world", choices=["world", "melspc"], type=str,
                        help="feature type")
    parser.add_argument("--n_quantize", default=256, type=int, help="number of quantization")
    parser.add_argument("--n_aux", default=28, type=int, help="number of dimension of aux feats")
    parser.add_argument("--n_resch", default=512, type=int, help="number of channels of residual output")
    parser.add_argument("--n_skipch", default=256, type=int, help="number of channels of skip output")
    parser.add_argument("--dilation_depth", default=10, type=int, help="depth of dilation")
    parser.add_argument("--dilation_repeat", default=1, type=int, help="number of repeating of dilation")
    parser.add_argument("--kernel_size", default=2, type=int, help="kernel size of dilated causal convolution")
    parser.add_argument("--upsampling_factor", default=80, type=int, help="upsampling factor of aux features")
    parser.add_argument("--use_upsampling_layer", default=True, type=_strtobool,
                        help="flag to use upsampling layer")
    parser.add_argument("--use_speaker_code", default=False, type=_strtobool, help="flag to use speaker code")
    parser.add_argument("--lr", default=1e-4, type=float, help="learning rate")
    parser.add_argument("--weight_decay", default=0.0, type=float, help="weight decay coefficient")
    parser.add_argument("--batch_length", default=20000, type=int, help="batch length (if set 0, utterance batch will be used)")
    parser.add_argument("--batch_size", default=1, type=int, help="batch size (if use utterance batch, batch_size will be 1.")
    parser.add_argument("--iters", default=200000, type=int, help="number of iterations")
    parser.add_argument("--checkpoint_interval", default=10000, type=int, help="how frequent saving model")
    parser.add_argument("--intervals", default=100, type=int, help="log interval")
    parser.add_argument("--seed", default=1, type=int, help="seed number")
    parser.add_argument("--resume", default=None, nargs="?", type=str, help="model path to restart training")
    parser.add_argument("--n_gpus", default=1, type=int, help="number of gpus")
    parser.add_argument("--verbose", default=1, type=int, help="log level")
    parser.add_argument("--math_mode", default="tf32", choices=["tf32", "fp32", "bf16"], type=str,
                        help="(H100 build) contraction precision of the training kernels; bf16 rounds the operands of "
                             "every product to bf16 (fp32 accumulation and storage) and needs a shape the composed "
                             "tensor-core path covers")
    parser.add_argument("--host_loader", default=False, type=_strtobool,
                        help="(H100 build) build the mini-batches on the host like the reference instead of on the GPU")
    parser.add_argument("--dev_waveforms", default=None, type=str, help="directory or list of held-out wav files")
    parser.add_argument("--dev_feats", default=None, type=str, help="directory or list of held-out aux feat files")
    parser.add_argument("--dev_interval", default=0, type=int,
                        help="log the held-out loss (utils/scoring.py) every this many iterations and at the end "
                             "(0: off)")
    parser.add_argument("--dev_batch_samples", default=1 << 19, type=int,
                        help="samples per held-out scoring batch (rows x longest row)")
    # (H100 build) the *-melspc recipes' stages 1-3 on the device, the corpus resident in HBM (utils/corpus.py); the
    # extraction flags are feature_extract.py's and noise_shaping.py's, with their defaults
    from pytorchwavenetvocoder_b200.bin.feature_extract import _optional_int
    parser.add_argument("--extract_features", default=False, type=_strtobool,
                        help="(H100 build) compute the melspc features, statistics (<expdir>/stats.h5) and optional "
                             "noise shaping from the raw wavs of --waveforms on the GPU and train from the resident "
                             "corpus, instead of reading --feats / --stats")
    parser.add_argument("--fs", default=16000, type=int, help="sampling frequency (--extract_features)")
    parser.add_argument("--shiftms", default=5, type=float, help="frame shift in msec (--extract_features)")
    parser.add_argument("--fftl", default=1024, type=int, help="FFT length (--extract_features)")
    parser.add_argument("--mspc_dim", default=80, type=int, help="dimension of mel spectrogram (--extract_features)")
    parser.add_argument("--fmin", default=None, nargs="?", type=_optional_int,
                        help="minimum frequency for melspc (empty: not given; --extract_features)")
    parser.add_argument("--fmax", default=None, nargs="?", type=_optional_int,
                        help="maximum frequency for melspc (empty: not given; --extract_features)")
    parser.add_argument("--highpass_cutoff", default=70, type=int,
                        help="cut off frequency of the low-cut filter, 0: none (--extract_features)")
    parser.add_argument("--noise_shaping", default=False, type=_strtobool,
                        help="train on noise-shaped wavs (noise_shaping.py --inv true; --extract_features)")
    parser.add_argument("--mcep_dim", default=24, type=int, help="dimension of mel cepstrum (--noise_shaping)")
    parser.add_argument("--mcep_alpha", default=0.41, type=float, help="alpha of mel cepstrum (--noise_shaping)")
    parser.add_argument("--mag", default=0.5, type=float, help="magnification of noise shaping (--noise_shaping)")
    return parser


def check_dev_args(args):
    """Refusals of the held-out flags, before anything is written: an error message, or None."""
    if (args.dev_waveforms is None) != (args.dev_feats is None):
        return "--dev_waveforms and --dev_feats go together"
    if args.dev_interval < 0:
        return "--dev_interval should be 0 (off) or a positive number of iterations, got %d" % args.dev_interval
    if args.dev_interval > 0 and args.dev_waveforms is None:
        return "--dev_interval %d needs --dev_waveforms and --dev_feats" % args.dev_interval
    if args.dev_batch_samples <= 0:
        return "--dev_batch_samples should be positive, got %d" % args.dev_batch_samples
    return None


def extract_wav_list(waveforms):
    """The wav files of --waveforms in the order train.py reads them: sorted from a directory, or the list's order."""
    if os.path.isdir(waveforms):
        return [waveforms + "/" + f for f in sorted(find_files(waveforms, "*.wav", use_dir_name=False))]
    if os.path.isfile(waveforms):
        return read_txt(waveforms)
    return None


def check_extract_args(args, parser):
    """Refusals of --extract_features, before any work: an error message, or None.  Reads the wav headers only."""
    from pytorchwavenetvocoder_b200.utils.corpus import wav_refusals
    from pytorchwavenetvocoder_b200.utils.melspc import shift_length
    if not args.extract_features:
        return None
    if args.feats is not None or args.stats is not None:
        return "--extract_features true computes the features and statistics: do not give --feats or --stats"
    if args.feature_type != "melspc":
        return "--extract_features true extracts melspc features: use --feature_type melspc"
    if args.mspc_dim != args.n_aux:
        return "--mspc_dim %d should equal --n_aux %d" % (args.mspc_dim, args.n_aux)
    if not args.use_upsampling_layer:
        return "--extract_features true trains with the up-sampling layer: --use_upsampling_layer false is not covered"
    hop = shift_length(args.shiftms, args.fs)
    if args.upsampling_factor != hop:
        return "--upsampling_factor %d should be the frame shift in samples, %d (--shiftms %g at --fs %d)" % (
            args.upsampling_factor, hop, args.shiftms, args.fs)
    if args.use_speaker_code:
        return "--extract_features true does not cover --use_speaker_code"
    if args.batch_length <= 0:
        return "--extract_features true covers the mini-batch mode: --batch_length 0 is not covered"
    if args.host_loader:
        return "--extract_features true trains from the device-resident corpus: --host_loader is not covered"
    for name in ("dev_waveforms", "dev_feats", "dev_interval", "dev_batch_samples"):
        if getattr(args, name) != parser.get_default(name):
            return "--extract_features true does not cover the held-out loss: do not give --%s" % name
    wav_list = extract_wav_list(args.waveforms)
    if wav_list is None:
        return "--waveforms should be directory or list."
    if len(wav_list) == 0:
        return "--waveforms names no wav files"
    bad = wav_refusals(wav_list, args.fs, args.fftl)
    if bad:
        return "; ".join(bad)
    return None


def file_generator(args, model, local):
    """The training generator over --waveforms / --feats with the --stats scaler: (generator, scaler)."""
    scaler = StandardScaler()
    scaler.mean_ = read_hdf5(args.stats, "/" + args.feature_type + "/mean")
    scaler.scale_ = read_hdf5(args.stats, "/" + args.feature_type + "/scale")
    wav_transform = lambda x: encode_mu_law(x, args.n_quantize)  # noqa: E731
    feat_transform = lambda x: scaler.transform(x)  # noqa: E731

    if os.path.isdir(args.waveforms):
        filenames = sorted(find_files(args.waveforms, "*.wav", use_dir_name=False))
        wav_list = [args.waveforms + "/" + filename for filename in filenames]
        feat_list = [args.feats + "/" + filename.replace(".wav", ".h5") for filename in filenames]
    elif os.path.isfile(args.waveforms):
        wav_list = read_txt(args.waveforms)
        feat_list = read_txt(args.feats)
    else:
        logging.error("--waveforms should be directory or list.")
        sys.exit(1)
    assert len(wav_list) == len(feat_list)
    logging.info("number of training data = %d." % len(wav_list))
    if args.batch_length > 0 and not args.host_loader:
        # mini-batch modes: windowing + mu-law + scaler on the device, utterances uploaded once (utils/device_loader.py);
        # same batches as train_generator below (tests/test_gpu_loader.py)
        from pytorchwavenetvocoder_b200.utils.device_loader import DeviceTrainGenerator
        generator = DeviceTrainGenerator(
            wav_list, feat_list, model.receptive_field, args.batch_length, args.batch_size,
            feature_type=args.feature_type, n_quantize=args.n_quantize, mean=scaler.mean_, scale=scaler.scale_,
            shuffle=True, upsampling_factor=args.upsampling_factor, use_upsampling_layer=args.use_upsampling_layer,
            use_speaker_code=args.use_speaker_code, device=local)
    else:
        generator = train_generator(
            wav_list, feat_list,
            receptive_field=model.receptive_field,
            batch_length=args.batch_length if args.batch_length > 0 else None,
            batch_size=args.batch_size,
            feature_type=args.feature_type,
            wav_transform=wav_transform,
            feat_transform=feat_transform,
            shuffle=True,
            upsampling_factor=args.upsampling_factor,
            use_upsampling_layer=args.use_upsampling_layer,
            use_speaker_code=args.use_speaker_code,
            device=local)
    return generator, scaler


def corpus_generator(args, model, rank, local):
    """--extract_features: the *-melspc recipes' stages 1-3 on this rank's GPU into a resident corpus, <expdir>/stats
    written by rank 0, and the generator over the corpus.  Every rank prepares the same corpus (the same bits)."""
    from pytorchwavenetvocoder_b200.bin.feature_extract import _feature_ext
    from pytorchwavenetvocoder_b200.utils.corpus import CorpusTooLarge, prepare_corpus
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceCorpusGenerator
    wav_list = extract_wav_list(args.waveforms)
    logging.info("number of training data = %d." % len(wav_list))
    try:
        corpus = prepare_corpus(wav_list, fs=args.fs, shiftms=args.shiftms, fftl=args.fftl, mspc_dim=args.mspc_dim,
                                fmin=args.fmin, fmax=args.fmax, highpass_cutoff=args.highpass_cutoff,
                                noise_shaping=args.noise_shaping, mcep_dim=args.mcep_dim,
                                mcep_alpha=args.mcep_alpha, mag=args.mag, device=local)
    except CorpusTooLarge as e:
        logging.error(str(e))
        sys.exit(1)
    if rank == 0:
        stats_file = args.expdir + "/stats" + _feature_ext()
        if os.path.exists(stats_file):
            os.remove(stats_file)                  # this run's statistics only
        corpus.write_stats(stats_file)
        logging.info("statistics written to %s." % stats_file)
    return DeviceCorpusGenerator(corpus, model.receptive_field, args.batch_length, args.batch_size,
                                 n_quantize=args.n_quantize, mean=corpus.mean, scale=corpus.scale, shuffle=True,
                                 device=local)


def dev_loss(model, utts, batch_samples):
    """Held-out loss of this rank's share ``utts`` gathered over ranks in list order (``parallel.gather_scores``):
    (Σ nll, Σ count, nats per sample), the same bits on any number of ranks.  Draws from no random generator."""
    from pytorchwavenetvocoder_b200.parallel import gather_scores
    from pytorchwavenetvocoder_b200.utils.scoring import corpus_mean, score_utterances
    nll, count = score_utterances(model, utts, batch_samples)
    return corpus_mean(*gather_scores(nll, count))


def _strtobool(v):
    if isinstance(v, bool):
        return v
    if str(v).lower() in ("y", "yes", "t", "true", "on", "1"):
        return True
    if str(v).lower() in ("n", "no", "f", "false", "off", "0"):
        return False
    raise argparse.ArgumentTypeError("invalid truth value %r" % v)


def main():
    """RUN TRAINING."""
    parser = get_parser()
    args = parser.parse_args()
    if not args.extract_features and (args.feats is None or args.stats is None):
        parser.error("the following arguments are required: %s" % ", ".join(
            f for f, v in (("--feats", args.feats), ("--stats", args.stats)) if v is None))
    fmt = '%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s'
    level = logging.INFO if args.verbose == 1 else (logging.DEBUG if args.verbose > 1 else logging.WARNING)
    logging.basicConfig(level=level, format=fmt, datefmt='%m/%d/%Y %I:%M:%S')
    if args.verbose < 1:
        logging.warning("logging is disabled.")
    for key, value in vars(args).items():
        logging.info("%s = %s" % (key, str(value)))

    refusal = check_extract_args(args, parser)
    if refusal is not None:
        logging.error(refusal)
        sys.exit(1)

    # one process per GPU (torchrun sets RANK / WORLD_SIZE / LOCAL_RANK)
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if args.n_gpus > 1 and "WORLD_SIZE" not in os.environ:
        # the recipes call `train.py --n_gpus N` as ONE process (reference nn.DataParallel, train.py:449-454); the
        # this build runs one process per GPU, so re-launch this command line under torch.distributed.run
        import socket
        with socket.socket() as s_:
            s_.bind(("127.0.0.1", 0))
            port = s_.getsockname()[1]
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.n_gpus),
               "--master-addr", "127.0.0.1", "--master-port", str(port), "-m", "pytorchwavenetvocoder_b200.bin.train"]
        logging.info("re-launching with one process per GPU: %s" % " ".join(cmd))
        os.execv(sys.executable, cmd + sys.argv[1:])
    if args.n_gpus > 1 and world != args.n_gpus:
        logging.error("--n_gpus %d but WORLD_SIZE is %d (launch with `torchrun --nproc-per-node %d`)."
                      % (args.n_gpus, world, args.n_gpus))
        sys.exit(1)
    refusal = check_dev_args(args)
    if refusal is not None:
        logging.error(refusal)
        sys.exit(1)
    if args.batch_length > 0 and args.batch_size % world != 0:
        # --batch_size stays the GLOBAL batch (the reference scatters one batch over the GPUs, train.py:449-454)
        logging.error("--batch_size %d is not divisible by the number of GPUs %d." % (args.batch_size, world))
        sys.exit(1)
    if not torch.cuda.is_available():
        logging.error("gpu is not available. please check the setting.")   # reference train.py:523-525
        sys.exit(1)
    torch.cuda.set_device(local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))

    if rank == 0 and not os.path.exists(args.expdir):
        os.makedirs(args.expdir)
    os.environ['PYTHONHASHSEED'] = str(args.seed)
    # every rank draws the SAME shuffles and therefore sees the same sequence of global batches; rank r trains on
    # rows [r*B/world, (r+1)*B/world) of each (torch.chunk order, like DataParallel's scatter)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    if rank == 0:
        torch.save(args, args.expdir + "/model.conf")

    upsampling_factor = args.upsampling_factor if args.use_upsampling_layer else 0
    model = WaveNet(
        n_quantize=args.n_quantize,
        n_aux=args.n_aux,
        n_resch=args.n_resch,
        n_skipch=args.n_skipch,
        dilation_depth=args.dilation_depth,
        dilation_repeat=args.dilation_repeat,
        kernel_size=args.kernel_size,
        upsampling_factor=upsampling_factor)
    logging.info(model)
    model.apply(initialize)
    model.train()
    from pytorchwavenetvocoder_b200.nets.wavenet import bf16_supported, tc_supported
    cfg_t = (args.n_quantize, args.n_aux, args.n_resch, args.n_skipch, args.dilation_depth, args.dilation_repeat,
             args.kernel_size, upsampling_factor)
    if args.math_mode == "bf16":
        if not bf16_supported(cfg_t):   # asked for explicitly: an error, not a quiet change of precision
            logging.error("--math_mode bf16 does not cover n_resch=%d n_skipch=%d n_aux=%d kernel_size=%d n_quantize=%d "
                          "(needs n_resch a multiple of 64, n_skipch / n_quantize multiples of 32 up to 256 or 512, "
                          "n_aux <= 256, kernel_size <= 3); use --math_mode tf32 or fp32"
                          % (args.n_resch, args.n_skipch, args.n_aux, args.kernel_size, args.n_quantize))
            sys.exit(1)
        model.math_mode = "bf16"
    else:
        model.math_mode = args.math_mode if (args.math_mode == "fp32" or tc_supported(cfg_t)) else "fp32"
    logging.info("math_mode = %s" % model.math_mode)

    model.cuda()   # before the optimizer: the fused (single multi-tensor kernel) Adam needs CUDA parameters
    # torch.optim.Adam (reference :457-460) with a one-launch step over the flat gradient buffer (optim.py); its
    # state_dict is torch's, so checkpoints stay interchangeable with the reference's
    from pytorchwavenetvocoder_b200.optim import Adam
    optimizer = Adam(model.parameters(), lr=args.lr, weight_decay=args.weight_decay, module=model)

    if args.extract_features:
        generator, scaler = corpus_generator(args, model, rank, local), None
    else:
        generator, scaler = file_generator(args, model, local)

    if args.resume is not None and len(args.resume) != 0:
        checkpoint = torch.load(args.resume, map_location=lambda storage, loc: storage, weights_only=False)
        iterations = checkpoint["iterations"]
        model.load_state_dict(checkpoint["model"])
        optimizer.load_state_dict(checkpoint["optimizer"])
        logging.info("restored from %d-iter checkpoint." % iterations)
    else:
        iterations = 0

    for state in optimizer.state.values():
        for key, value in state.items():
            if torch.is_tensor(value):
                state[key] = value.cuda()
    sync = None
    if world > 1:
        from pytorchwavenetvocoder_b200.parallel import GradAllReduce
        sync = GradAllReduce(model)

    dev_utts = None
    if args.dev_interval > 0:
        # this rank's np.array_split share of the held-out list, aligned once (utils/scoring.py); scoring it draws from
        # no random generator and leaves the training generator alone, so the checkpoints do not change
        from pytorchwavenetvocoder_b200.bin.evaluate import file_lists
        from pytorchwavenetvocoder_b200.parallel import shard_utterances
        from pytorchwavenetvocoder_b200.utils.scoring import load_utterance
        dev_wavs, dev_feats = file_lists(args.dev_waveforms, args.dev_feats)
        dev_utts = [load_utterance(w, f, args, scaler) for w, f in
                    zip(shard_utterances(dev_wavs, world, rank), shard_utterances(dev_feats, world, rank))]
        logging.info("number of held-out data = %d." % len(dev_wavs))

    def log_dev(it):
        s_, n_, mean = dev_loss(model, dev_utts, args.dev_batch_samples)
        if rank == 0:
            logging.info("(iter:%d) dev loss = %.6f (%d samples)" % (it, mean, n_))

    loss = torch.zeros((), device="cuda")    # summed on the device: no host sync per step (reference :540 syncs)
    total = 0
    debug = logging.getLogger().isEnabledFor(logging.DEBUG)
    for i in range(iterations, args.iters):
        start = time.time()
        (batch_x, batch_h), batch_t = generator.next()
        if world > 1 and batch_x.size(0) > 1:
            per = batch_x.size(0) // world
            batch_x, batch_h, batch_t = (v[rank * per:(rank + 1) * per].contiguous() for v in (batch_x, batch_h, batch_t))
        # = cross_entropy(model(batch_x, batch_h), batch_t, rf): CE on [:, receptive_field:] (reference :533-536)
        batch_loss = model.forward_loss(batch_x, batch_h, batch_t, model.receptive_field)
        optimizer.zero_grad()
        batch_loss.backward()
        if sync is not None:
            sync.allreduce()
        optimizer.step()
        loss += batch_loss.detach()
        total += time.time() - start
        if debug:
            logging.debug("batch loss = %.3f (%.3f sec / batch)" % (batch_loss.item(), time.time() - start))

        if (i + 1) % args.intervals == 0:
            loss_sum = float(loss)
            if world > 1:   # equal per-rank batches: the global mean is the mean of the rank means
                lt = loss.clone()
                torch.distributed.all_reduce(lt)
                loss_sum = float(lt) / world
            loss.zero_()
            logging.info("(iter:%d) average loss = %.6f (%.3f sec / batch)" % (
                i + 1, loss_sum / args.intervals, total / args.intervals))
            remain = int((args.iters - (i + 1)) * (total / args.intervals))
            logging.info("estimated required time = %02d:%02d:%02d:%02d" % (
                remain // 86400, remain % 86400 // 3600, remain % 3600 // 60, remain % 60))
            total = 0

        if (i + 1) % args.checkpoint_interval == 0 and rank == 0:
            save_checkpoint(args.expdir, model, optimizer, i + 1)
        if dev_utts is not None and (i + 1) % args.dev_interval == 0:
            log_dev(i + 1)

    if dev_utts is not None and (args.iters <= iterations or args.iters % args.dev_interval != 0):
        log_dev(max(args.iters, iterations))
    if rank == 0:
        torch.save({"model": model.state_dict()}, args.expdir + "/checkpoint-final.pkl")
        logging.info("final checkpoint created.")
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
