# -*- coding: utf-8 -*-
"""GPU tier: resumable MLSA filtering (wnb_mlsa_filter_state, MlsaStreamFilter, bin/decode.py --noise_shaping).

Signals cut into consecutive chunks, filtered chunk by chunk and concatenated must equal ``mlsa_filter_batch`` of the
whole signal and the C oracle (oracle/mlsa_oracle.c) bit for bit, int16 and float64:
* pd 4 and 5, orders 2, 24 (the recipes' 25 coefficients) and 59, +coef and -coef;
* chunks of 1, 7, 8, 9 and 80 samples, random sizes with zeros, one chunk holding everything; lengths 0 .. 3 001;
* launches whose 4 segments per warp have very different lengths (a state stored at the warp's end fails here);
* a closed key's slot reused by a new signal, a new key whose first chunk is empty, a state table that grows.
End to end: a decode session's ``step_pcm16`` chunks (64/512 on the warp decoder, arctic 512/256 on the bf16 decoder)
and a decode pool's per-stream chunks, filtered as they arrive, equal one-shot decoding followed by whole-signal
filtering; ``bin/decode.py --noise_shaping`` (with and without ``--chunk_frames``) writes the bytes of ``bin/decode.py``
followed by ``bin/noise_shaping.py --inv false``."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mlsa_oracle as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENGTHS = [0, 1, 7, 8, 9, 15, 80, 81, 1000, 3001]


def _coef(rng, order, alpha):
    return M.convert_mcep_to_mlsa_coef(rng.randn(order + 1) * 0.6, 0.5, alpha)


def _signals(rng, lengths, i16):
    xs = []
    for n in lengths:
        x = np.cumsum(rng.randn(n))
        x = x / (np.abs(x).max() + 1e-9) * 9000.0 + rng.randn(n) * 20.0 if n > 1 else rng.randn(n) * 100
        xs.append(np.int16(x) if i16 else x)
    return xs


def _schedule(kind, n, rng):
    """chunk sizes covering n samples"""
    if kind == "whole":
        return [n]
    if kind == "random":
        out = []
        while sum(out) < n:
            out.append(int(rng.choice([0, 0, 1, 2, 5, 8, 13, 64, 200, 777])))
        return out
    return [kind] * ((n + kind - 1) // kind)


def _run_chunked(filt, xs, schedules, device="cuda"):
    """feed signal k's chunks under key k, one call per round (a finished signal drops out), -> concatenated outputs"""
    pos = [0] * len(xs)
    got = [[] for _ in xs]
    for r in range(max(len(s) for s in schedules)):
        chunks = {}
        for k, (x, s) in enumerate(zip(xs, schedules)):
            if r < len(s):
                c = x[pos[k]:pos[k] + s[r]]          # the last chunk of a schedule may run past the end
                chunks[k] = torch.from_numpy(np.ascontiguousarray(c)).to(device)
                pos[k] += len(c)
        for k, y in filt.filter(chunks).items():
            got[k].append(y.cpu().numpy())
    assert pos == [len(x) for x in xs]
    return [np.concatenate(g) if g else np.zeros(0, dtype=x.dtype) for g, x in zip(got, xs)]


def _oracle(x, coef, alpha, pd):
    """the oracle's recursion; int16 in: np.float64 in, np.int16 out (noise_shaping_one, which needs 2+ samples)"""
    y = M.filter_const(x.astype(np.float64), coef, alpha, pd)
    return M.to_int16(y) if x.dtype == np.int16 else y


@pytest.mark.parametrize("i16", [True, False])
@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("order,alpha,pd", [(24, 0.41, 4), (24, 0.41, 5), (59, 0.455, 4), (2, 0.35, 5)])
def test_chunked_equals_whole(order, alpha, pd, sign, i16):
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter, mlsa_filter_batch
    rng = np.random.RandomState(order * 10 + pd)
    coef = sign * _coef(rng, order, alpha)
    xs = _signals(rng, LENGTHS, i16)
    whole = mlsa_filter_batch(xs, coef, alpha, pd=pd)
    for x, w in zip(xs, whole):
        assert np.array_equal(w, _oracle(x, coef, alpha, pd))
    for kind in (1, 7, 8, 9, 80, "random", "whole"):
        filt = MlsaStreamFilter(coef, alpha, pd)
        got = _run_chunked(filt, xs, [_schedule(kind, len(x), rng) for x in xs])
        for k, (g, w) in enumerate(zip(got, whole)):
            assert g.dtype == w.dtype and np.array_equal(g, w), (kind, LENGTHS[k])


def test_segments_of_one_warp_with_different_lengths():
    """every call puts chunks of very different lengths (0 .. 1 500) side by side in the 4 segments of a warp, so the
    short ones run on past their end inside the launch; their carried state must be the one after their own end"""
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter, mlsa_filter_batch
    rng = np.random.RandomState(3)
    coef = _coef(rng, 24, 0.41)
    sizes = [0, 1, 3, 8, 9, 31, 517, 1500]
    schedules = [[int(rng.choice(sizes)) for _ in range(12)] for _ in range(11)]
    schedules[0] = [1500, 1] * 6          # row 0: alternately the longest and the shortest of its warp
    schedules[1] = [1, 1500] * 6
    xs = _signals(rng, [sum(s) for s in schedules], True)
    got = _run_chunked(MlsaStreamFilter(coef, 0.41, 4), xs, schedules)
    for g, w in zip(got, mlsa_filter_batch(xs, coef, 0.41)):
        assert np.array_equal(g, w)


def test_closed_key_reused_and_empty_first_chunk():
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter, mlsa_filter_batch
    rng = np.random.RandomState(4)
    coef = _coef(rng, 24, 0.41)
    a, b, c = _signals(rng, [900, 700, 500], False)
    want_b, want_c = mlsa_filter_batch([b, c], coef, 0.41)
    f = MlsaStreamFilter(coef, 0.41, 4)
    dev = lambda v: torch.from_numpy(np.ascontiguousarray(v)).cuda()   # noqa: E731
    f.filter({"a": dev(a[:400])})
    slot = f.slot("a")
    f.close("a")                                      # "a" leaves a non-zero state in its slot
    # "b" takes the slot with an empty first chunk beside a non-empty one: it must still start from zero later
    out = f.filter({"b": dev(b[:0]), "c": dev(c[:250])})
    assert f.slot("b") == slot and out["b"].numel() == 0
    got_b = [f.filter({"b": dev(b[i:i + 70]), "c": dev(c[250 + i:250 + i + 70])}) for i in range(0, 700, 70)]
    assert np.array_equal(np.concatenate([g["b"].cpu().numpy() for g in got_b]), want_b)
    assert np.array_equal(np.concatenate([out["c"].cpu().numpy()] + [g["c"].cpu().numpy() for g in got_b]), want_c)
    # a table that grows while keys hold state: 130 signals, new keys arriving over the calls
    xs = _signals(rng, [int(v) for v in rng.randint(100, 400, size=130)], True)
    schedules = [[0] * (k // 20) + _schedule(37, len(x), rng) for k, x in enumerate(xs)]
    got = _run_chunked(f, xs, schedules)
    for g, w in zip(got, mlsa_filter_batch(xs, coef, 0.41)):
        assert np.array_equal(g, w)


# ---- decode sessions and pools -------------------------------------------------------------------------------------
def _session_case(shape, decode_math, B, max_n, seed):
    from tests.test_gpu_decode_session import _inputs, _model
    cfg, net = _model(shape, decode_math)
    x, h, n_list = _inputs(cfg, B, 1, max_n, seed)
    return cfg, net, x, h, n_list


@pytest.mark.parametrize("case", ["warp_64_512", "bf16_arctic"])
def test_session_chunks_filtered_equal_one_shot(case):
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter, mlsa_filter_batch
    from tests.test_gpu_decode_session import BENCH
    if case == "warp_64_512":
        cfg, net, x, h, n_list = _session_case(BENCH, "fp32", 5, 700, 1)
        kernel = "warp"
    else:
        cfg, net, x, h, n_list = _session_case((256, 28, 512, 256, 10, 3, 2, 80), "bf16", 3, 500, 2)
        kernel = "bf16"
    rng = np.random.RandomState(5)
    coef = _coef(rng, 24, 0.41)
    torch.manual_seed(11)
    with torch.no_grad():
        pcm = net.batch_fast_generate_pcm16(x, h, n_list)
    order = sorted(range(len(n_list)), key=lambda b: (n_list[b], b))
    want = dict(zip(order, mlsa_filter_batch(pcm, coef, 0.41)))
    for sched in ("ones", "random"):
        torch.manual_seed(11)
        sess = net.decode_session(x, n_list)
        assert sess.kernel == kernel
        filt = MlsaStreamFilter(coef, 0.41, 4)
        got = {b: [] for b in range(len(n_list))}
        f0 = 0
        while not sess.done:
            F = 1 if sched == "ones" else int(rng.randint(1, 6))
            out = sess.step_pcm16(h[:, :, f0:f0 + F])
            f0 += F
            for b, y in filt.filter({b: out[b, :c] for b, c in enumerate(sess.last_counts)}).items():
                got[b].append(y.cpu().numpy())
        for b in range(len(n_list)):
            assert np.array_equal(np.concatenate(got[b]), want[b]), (case, sched, b)


def test_pool_streams_filtered_equal_one_shot():
    from pytorchwavenetvocoder_b200.nets.wavenet import codes_to_pcm16
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter, mlsa_filter_batch
    from tests.test_gpu_decode_pool import SHALLOW_256, _model, _one_shot, _streams
    cfg, net = _model(SHALLOW_256)
    streams = _streams(cfg, 24, 31)
    codes = _one_shot(net, streams, "sampling", 8)
    coef = _coef(np.random.RandomState(6), 24, 0.41)
    want = mlsa_filter_batch([codes_to_pcm16(codes[k].cuda(), 256).cpu().numpy() for k in range(len(streams))], coef,
                             0.41)
    rng = np.random.RandomState(9)
    pool = net.decode_pool(8, "sampling", 8)
    filt = MlsaStreamFilter(coef, 0.41, 4)
    got = {k: [] for k in range(len(streams))}
    sent = [0] * len(streams)
    it = 0
    while it <= max(a for _, _, _, a in streams) or not all(pool.finished(k) for k in range(len(streams))):
        for k, (x, total, h, arrival) in enumerate(streams):
            if arrival == it:
                pool.admit(x, total, h[:, :2], stream=k)
                sent[k] = 2
            elif arrival < it and not pool.finished(k) and sent[k] < h.size(1):
                F = min(int(rng.randint(0, 30)), h.size(1) - sent[k])
                pool.feed(k, h[:, sent[k]:sent[k] + F])
                sent[k] += F
        it += 1
        for k, y in filt.filter(pool.step_pcm16(int(rng.randint(1, 120)))).items():
            got[k].append(y.cpu().numpy())
            if pool.finished(k):
                filt.close(k)
    for k in range(len(streams)):
        assert np.array_equal(np.concatenate(got[k]), want[k]), k


# ---- bin/decode.py --noise_shaping ---------------------------------------------------------------------------------
def _cli(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", module] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=600)
    assert r.returncode == 0, r.stdout.decode()[-3000:]


def test_cli_noise_shaping_equals_decode_then_restore(tmp_path):
    """decode.py --noise_shaping (one-shot and --chunk_frames 7, batch and single-utterance mode) writes the bytes of
    decode.py followed by noise_shaping.py --inv false.  The decoder's wav files are written by our PCM_16 writer here:
    with soundfile installed, decode.py without the flag quantises in libsndfile instead (see bin/decode.py)."""
    from pytorchwavenetvocoder_b200.nets import WaveNet
    from pytorchwavenetvocoder_b200.utils import have_soundfile, write_hdf5
    if have_soundfile():
        pytest.skip("the byte equality is the pipeline's with our PCM_16 writer (soundfile absent)")
    U, D_ = 16, 28
    rng = np.random.RandomState(8)
    torch.manual_seed(0)
    net = WaveNet(256, D_, 64, 128, 3, 2, 2, U)
    expdir, featdir = tmp_path / "exp", tmp_path / "feats"
    expdir.mkdir()
    featdir.mkdir()
    torch.save({"model": net.state_dict()}, str(expdir / "checkpoint-final.pkl"))
    conf = argparse.Namespace(n_quantize=256, n_aux=D_, n_resch=64, n_skipch=128, dilation_depth=3, dilation_repeat=2,
                              kernel_size=2, upsampling_factor=U, use_upsampling_layer=True, feature_type="world",
                              use_speaker_code=False)
    torch.save(conf, str(expdir / "model.conf"))
    feats = []
    for i, nf in enumerate([40, 66, 53]):
        f = str(featdir / ("c%d.npz" % i))
        write_hdf5(f, "/world", rng.standard_normal((nf, D_)))
        feats.append(f)
    fl, stats = str(tmp_path / "feats.scp"), str(tmp_path / "stats.npz")
    open(fl, "w").write("\n".join(feats) + "\n")
    write_hdf5(stats, "/world/mean", np.zeros(D_))
    write_hdf5(stats, "/world/scale", np.ones(D_))
    write_hdf5(stats, "/mlsa/coef", M.convert_mcep_to_mlsa_coef(rng.randn(25) * 0.5, 0.5, 0.41))
    write_hdf5(stats, "/mlsa/alpha", 0.41)
    for bs in ("3", "1"):
        common = ["--feats", fl, "--checkpoint", str(expdir / "checkpoint-final.pkl"), "--stats", stats, "--fs", "16000",
                  "--batch_size", bs, "--intervals", "100", "--seed", "5"]
        plain, restored = str(tmp_path / ("plain%s" % bs)), str(tmp_path / ("restored%s" % bs))
        _cli("pytorchwavenetvocoder_b200.bin.decode", common + ["--outdir", plain])
        _cli("pytorchwavenetvocoder_b200.bin.noise_shaping", ["--waveforms", plain, "--stats", stats, "--outdir",
                                                              restored, "--fs", "16000", "--inv", "false"])
        for chunk in ("0", "7"):
            od = str(tmp_path / ("ns_bs%s_c%s" % (bs, chunk)))
            _cli("pytorchwavenetvocoder_b200.bin.decode", common + ["--outdir", od, "--noise_shaping",
                                                                    "--chunk_frames", chunk])
            for i in range(3):
                want = open(os.path.join(restored, "c%d.wav" % i), "rb").read()
                got = open(os.path.join(od, "c%d.wav" % i), "rb").read()
                assert len(want) > 44 and got == want, (bs, chunk, i)
                assert got != open(os.path.join(plain, "c%d.wav" % i), "rb").read()
