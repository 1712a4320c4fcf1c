# -*- coding: utf-8 -*-
"""CPU tier of the device-resident corpus (utils/corpus.py, utils/device_loader.DeviceCorpusGenerator,
``bin/train.py --extract_features``): the epoch table and its binary search against a restatement of the ring loader's
bookkeeping, the trimming and resident-size arithmetic and its refusal, and every refusal of ``--extract_features``."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ring_positions(orders, lengths):
    """(stream start, utterance, length) of every utterance DeviceTrainGenerator._append puts in its ring, epoch after
    epoch: an empty utterance is skipped, every other one starts at the running tail"""
    tail, out = 0, []
    for order in orders:
        for u in order:
            n = int(lengths[u])
            if n == 0:
                continue
            out.append((tail, u, n))
            tail += n
    return out


@pytest.mark.parametrize("seed", range(40))
def test_epoch_table_maps_every_stream_position(seed):
    from pytorchwavenetvocoder_b200.utils.device_loader import corpus_index, corpus_table
    rng = np.random.RandomState(seed)
    U = int(rng.choice([1, 80, 256]))
    N = rng.randint(1, 9)
    # whole frames, some empty, some shorter than a hop of a few frames
    lengths = (rng.randint(0, 7, N) * rng.choice([0, 1, 1, 1], N) * U).astype(np.int64)
    if lengths.sum() == 0:
        lengths[rng.randint(N)] = U
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    n_epochs = rng.randint(1, 6)
    order, orders = np.arange(N), []
    for _ in range(n_epochs + 3):
        order = order[rng.permutation(N)]
        orders.append(order)
    L = int(lengths.sum())
    ring = _ring_positions(orders, lengths)
    want = np.empty(len(orders) * L, dtype=np.int64)
    for start, u, n in ring:
        want[start:start + n] = offsets[u] + np.arange(n)
    for e0 in range(len(orders)):
        for e1 in range(e0, min(e0 + n_epochs, len(orders))):
            starts, offs, begin, end = corpus_table(orders[e0:e1 + 1], e0, lengths, offsets)
            assert begin == e0 * L and end == (e1 + 1) * L
            assert np.all(np.diff(starts) > 0) and len(starts) == (e1 - e0 + 1) * np.count_nonzero(lengths)
            assert np.all(offs % U == 0) and np.all(starts % U == 0)
            p = np.arange(begin, end, dtype=np.int64)
            got = corpus_index(starts, offs, p)
            assert np.array_equal(got, want[begin:end]), (e0, e1)
            # frame rows: the row of the frame's first sample, what the kernel reads
            f = np.arange(begin // U, end // U, dtype=np.int64)
            assert np.array_equal(corpus_index(starts, offs, f * U) // U, want[f * U] // U)


@pytest.mark.parametrize("n", [1, 79, 80, 81, 159, 160, 161, 1023, 1024, 16000, 16001, 123457])
@pytest.mark.parametrize("U", [80, 256, 110])
def test_trimmed_length_is_load_pair_frames(tmp_path, n, U):
    """trimmed_length equals what load_pair_frames keeps of a wav and its 1 + n // U frames (up-sampling mode)"""
    from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav
    from pytorchwavenetvocoder_b200.utils.corpus import trimmed_length
    from pytorchwavenetvocoder_b200.utils.device_loader import load_pair_frames
    w, f = str(tmp_path / "a.wav"), str(tmp_path / "a.npz")
    write_wav(w, np.zeros(n), 16000)
    write_hdf5(f, "/melspc", np.zeros((1 + n // U, 3), np.float32))
    x, h = load_pair_frames(w, f, "melspc", U, True, False)
    assert trimmed_length(n, U) == (len(x), len(h))


def test_resident_size_and_refusal():
    from pytorchwavenetvocoder_b200.utils.corpus import FILE_PIPELINE, fit_refusal, resident_bytes, trimmed_length
    ns = [16000, 1023, 50000, 80 * 7]
    U, D = 80, 80
    want = sum(2 * trimmed_length(n, U)[0] + 4 * D * trimmed_length(n, U)[1] for n in ns)
    assert want == 2 * (15920 + 960 + 49920 + 480) + 4 * D * (199 + 12 + 624 + 6)
    assert resident_bytes(ns, U, D) == want
    assert fit_refusal(want, 2 * want) is None
    assert fit_refusal(want, 2 * want + 1) is None
    msg = fit_refusal(want, 2 * want - 2)
    assert msg is not None and str(want) in msg and str(want - 1) in msg and FILE_PIPELINE in msg
    # LJSpeech-sized: about 1.9 G samples of 22.05 kHz at a 256-sample hop, 80 mels
    lj = [190000] * 10000
    assert abs(resident_bytes(lj, 256, 80) - (3.8e9 + 2.4e9)) < 0.05e9


# ---- bin/train.py --extract_features refusals -------------------------------------------------------------------
@pytest.fixture(scope="module")
def wavs(tmp_path_factory):
    from pytorchwavenetvocoder_b200.utils import write_wav_int16
    root = tmp_path_factory.mktemp("wavs")
    good = root / "good"
    good.mkdir()
    for i, n in enumerate([3000, 1024, 5000]):
        write_wav_int16(str(good / ("g%d.wav" % i)), 16000, np.int16(np.arange(n) % 300))
    rate = root / "rate"
    rate.mkdir()
    write_wav_int16(str(rate / "a.wav"), 16000, np.zeros(3000, np.int16))
    write_wav_int16(str(rate / "b.wav"), 22050, np.zeros(3000, np.int16))
    short = root / "short"
    short.mkdir()
    write_wav_int16(str(short / "a.wav"), 16000, np.zeros(3000, np.int16))
    write_wav_int16(str(short / "b.wav"), 16000, np.zeros(1023, np.int16))
    return str(good), str(rate), str(short)


REFUSALS = {
    "feats": (["--feats", "f.scp"], "do not give --feats or --stats"),
    "stats": (["--stats", "s.h5"], "do not give --feats or --stats"),
    "feature_type": (["--feature_type", "world"], "use --feature_type melspc"),
    "mspc_dim": (["--mspc_dim", "40"], "--mspc_dim 40 should equal --n_aux 80"),
    "no_upsampling_layer": (["--use_upsampling_layer", "false"], "--use_upsampling_layer false is not covered"),
    "upsampling_factor": (["--upsampling_factor", "160"], "--upsampling_factor 160 should be the frame shift in samples, 80"),
    "shift": (["--shiftms", "10"], "--upsampling_factor 80 should be the frame shift in samples, 160"),
    "speaker_code": (["--use_speaker_code", "true"], "does not cover --use_speaker_code"),
    "utterance_batch": (["--batch_length", "0"], "--batch_length 0 is not covered"),
    "host_loader": (["--host_loader", "true"], "--host_loader is not covered"),
    "dev_waveforms": (["--dev_waveforms", "d.scp"], "do not give --dev_waveforms"),
    "dev_feats": (["--dev_feats", "d.scp"], "do not give --dev_feats"),
    "dev_interval": (["--dev_interval", "5"], "do not give --dev_interval"),
    "dev_batch_samples": (["--dev_batch_samples", "1000"], "do not give --dev_batch_samples"),
    "sampling_rate": ("rate", "b.wav: sampling rate 22050, not --fs 16000"),
    "shorter_than_fftl": ("short", "b.wav has 1023 samples, fewer than fftl = 1024"),
}


def _argv(wavs, case):
    good, rate, short = wavs
    extra, _ = REFUSALS[case]
    wavdir = {"rate": rate, "short": short}.get(extra, good) if isinstance(extra, str) else good
    return (["--waveforms", wavdir, "--expdir", "exp", "--extract_features", "true", "--feature_type", "melspc",
             "--n_aux", "80"] + (extra if isinstance(extra, list) else []))


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_extract_features_refusals(wavs, case):
    from pytorchwavenetvocoder_b200.bin.train import check_extract_args, get_parser
    parser = get_parser()
    msg = check_extract_args(parser.parse_args(_argv(wavs, case)), parser)
    assert msg is not None and REFUSALS[case][1] in msg, msg


def test_extract_features_accepts_the_recipe_flags(wavs):
    from pytorchwavenetvocoder_b200.bin.train import check_extract_args, get_parser
    parser = get_parser()
    args = parser.parse_args(_argv(wavs, "feats")[:-2] + ["--fmin", "", "--fmax", "", "--noise_shaping", "true",
                                                         "--mcep_dim", "25", "--mcep_alpha", "0.410", "--mag", "0.5"])
    assert check_extract_args(args, parser) is None
    assert args.fmin is None and args.fmax is None and args.noise_shaping and args.mcep_dim == 25
    # without --extract_features nothing is checked
    args = parser.parse_args(["--waveforms", "w", "--feats", "f", "--stats", "s", "--expdir", "e"])
    assert check_extract_args(args, parser) is None and not args.extract_features


@pytest.mark.parametrize("case", ["feats", "shorter_than_fftl"])
def test_train_exits_before_touching_a_gpu(wavs, case, tmp_path):
    """the command exits 1 with the message, with no GPU visible and before it creates --expdir"""
    argv = _argv(wavs, case)
    argv[argv.index("--expdir") + 1] = str(tmp_path / "exp")
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.train"] + argv, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=300)
    out = r.stdout.decode()
    assert r.returncode == 1 and REFUSALS[case][1] in out, out[-2000:]
    assert "gpu is not available" not in out and not os.path.exists(str(tmp_path / "exp"))


def test_train_still_requires_feats_and_stats_without_the_flag(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.train", "--waveforms", "w", "--feats", "f",
                        "--expdir", str(tmp_path)], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=300)
    assert r.returncode == 2 and "the following arguments are required: --stats" in r.stdout.decode()
