# -*- coding: utf-8 -*-
"""GPU tier: streaming mel-spectrogram extraction (wnb_melspc_stream, MelspcStream, bin/resynthesize.py).

Every comparison is exact (torch.equal / np.array_equal):
* a key's frames, concatenated, equal ``melspc_batch`` of its whole signal: lengths 1, 2, half, half + 1, fftl and 10 s,
  int16 and float64, cutoff 0 and 70, fftl 64 / 1024 / 4096 with hops 80 / 110 / 256, chunks of 1, hop +- 1, half,
  half + 1, fftl and random sizes with empty chunks, many keys per call, 1024 keys in one call, closed and reused slots;
* the scaled output equals ``StandardScaler.transform`` arithmetic of both scaler modes on the raw features;
* at most 2 launches per call, none for an empty call, and two runs are bit-identical;
* a decode session and a bf16 decode pool fed by the stream decode the codes of one-shot decoding of the
  ``melspc_batch`` features;
* ``bin/resynthesize.py`` writes the bytes of ``feature_extract.py --feature_type melspc`` + ``decode.py``."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pytorchwavenetvocoder_b200 import _lib
from pytorchwavenetvocoder_b200.utils.melspc import MelspcStream, melspc_batch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _signals(rng, lengths, i16):
    xs = []
    for n in lengths:
        x = np.cumsum(rng.randn(n)) * 300 + rng.randn(n) * 2000
        x = np.clip(x, -32768, 32767)
        xs.append(np.int16(x) if i16 else np.round(x * 8) / 8)
    return xs


def _sizes(kind, n, fftl, hop, rng):
    half = fftl // 2
    if kind == "whole":
        return [n]
    if kind == "random":
        out = []
        while sum(out) < n:
            out.append(int(rng.choice([0, 0, 1, 2, hop, 333, fftl, 3 * fftl, 20000])))
        return out
    step = {"one": 1, "hop-1": max(hop - 1, 1), "hop+1": hop + 1, "half": half, "half+1": half + 1, "fftl": fftl}[kind]
    if n > 40000 and step < 64:
        step = 1600           # keep the 10 s signals to a few hundred calls
    return [step] * ((n + step - 1) // step)


def _run(stream, xs, schedules, dev="cuda"):
    """push signal k's chunks under key k, one call per round; a key ends in the call of its last chunk"""
    got = [[] for _ in xs]
    pos = [0] * len(xs)
    for r in range(max(len(s) for s in schedules)):
        chunks, final = {}, []
        for k, (x, s) in enumerate(zip(xs, schedules)):
            if r >= len(s):
                continue
            chunks[k] = torch.from_numpy(x[pos[k]:pos[k] + s[r]]).to(dev)
            pos[k] += s[r]
            if r == len(s) - 1:
                final.append(k)
        for k, v in stream.push(chunks, final).items():
            got[k].append(v)
    return [torch.cat(g, 1 if stream._mean is not None else 0) for g in got]


@pytest.mark.parametrize("fftl,hop", [(64, 80), (1024, 80), (1024, 110), (4096, 256)])
@pytest.mark.parametrize("cutoff", [0, 70])
@pytest.mark.parametrize("i16", [True, False])
def test_stream_equals_batch(fftl, hop, cutoff, i16):
    fs = 16000
    rng = np.random.RandomState(fftl + hop + cutoff + i16)
    half = fftl // 2
    lengths = [1, 2, half, half + 1, fftl, 160000]
    xs = _signals(rng, lengths, i16)
    want = melspc_batch(xs, fs, fftl, hop, 80, highpass_cutoff=cutoff)
    for kinds in (["one", "hop-1", "hop+1", "half", "half+1", "fftl"], ["random"] * 6, ["whole"] * 6):
        s = MelspcStream(fs, fftl, hop, 80, highpass_cutoff=cutoff)
        sched = [_sizes(k, len(x), fftl, hop, rng) for k, x in zip(kinds, xs)]
        got = _run(s, xs, sched)
        for i in range(len(xs)):
            assert np.array_equal(got[i].cpu().numpy(), want[i]), (kinds[i], lengths[i])


def test_many_keys_reuse_and_1024_keys():
    fs, fftl, hop = 16000, 1024, 80
    rng = np.random.RandomState(3)
    s = MelspcStream(fs, fftl, hop, 80, highpass_cutoff=70, fmin=80, fmax=7600)
    # 1024 keys in one call, each its whole signal, lengths 1 .. 3000
    xs = _signals(rng, rng.randint(1, 3000, 1024), True)
    out = s.push({k: torch.from_numpy(x).cuda() for k, x in enumerate(xs)}, final=range(1024))
    want = melspc_batch(xs, fs, fftl, hop, 80, fmin=80, fmax=7600, highpass_cutoff=70)
    assert all(np.array_equal(out[k].cpu().numpy(), want[k]) for k in range(1024))
    assert s.slot(0) is None
    # keys that end at different times, slots reused by new keys, a closed key, empty chunks
    xs = _signals(rng, rng.randint(1, 6000, 40), True)
    want = melspc_batch(xs, fs, fftl, hop, 80, fmin=80, fmax=7600, highpass_cutoff=70)
    got = {k: [] for k in range(40)}
    pos = {k: 0 for k in range(40)}
    live, nxt = set(range(10)), 10
    s.push({"gone": torch.from_numpy(xs[0][:700]).cuda()})
    s.close("gone")
    while live:
        chunks, final = {}, []
        for k in sorted(live):
            n = int(rng.choice([0, 0, 1, 79, 81, 512, 513, 1600]))
            chunks[k] = torch.from_numpy(xs[k][pos[k]:pos[k] + n]).cuda()
            pos[k] += chunks[k].numel()
            if pos[k] == len(xs[k]):
                final.append(k)
        for k, v in s.push(chunks, final).items():
            got[k].append(v)
        for k in final:
            live.discard(k)
            if nxt < 40:
                live.add(nxt)
                nxt += 1
    for k in range(40):
        assert np.array_equal(torch.cat(got[k]).cpu().numpy(), want[k]), k


@pytest.mark.parametrize("mode", [0, 2])
def test_scaled_output(mode):
    fs, fftl, hop = 16000, 1024, 80
    rng = np.random.RandomState(mode)
    xs = _signals(rng, [5000, 12000, 300], True)
    mean, scale = rng.randn(80) * 2 - 4, 0.3 + rng.rand(80)
    raw = melspc_batch(xs, fs, fftl, hop, 80, highpass_cutoff=70)
    s = MelspcStream(fs, fftl, hop, 80, highpass_cutoff=70, scaler=(mean, scale), scaler_mode=mode)
    got = _run(s, xs, [_sizes("random", len(x), fftl, hop, rng) for x in xs])
    for f, g in zip(raw, got):
        if mode == 0:
            want = ((f.astype(np.float64) - mean).astype(np.float32).astype(np.float64) / scale).astype(np.float32)
        else:
            want = (f - mean.astype(np.float32)) / scale.astype(np.float32)
        assert g.shape == (80, len(f)) and np.array_equal(g.cpu().numpy(), want.T)
    from sklearn.preprocessing import StandardScaler
    from pytorchwavenetvocoder_b200.utils.device_loader import _f32_scaler_mode
    if _f32_scaler_mode() == mode:
        sc = StandardScaler()
        sc.mean_, sc.scale_ = mean, scale
        for f, g in zip(raw, got):
            assert np.array_equal(g.cpu().numpy(), sc.transform(f).T)


def test_launch_counts_and_determinism():
    fs, fftl, hop = 16000, 1024, 80
    rng = np.random.RandomState(9)
    xs = _signals(rng, [9000, 4000, 777], True)
    sched = [_sizes("random", len(x), fftl, hop, rng) for x in xs]
    runs = []
    for _ in range(2):
        s = MelspcStream(fs, fftl, hop, 80, highpass_cutoff=70)
        c0 = _lib.launch_count()
        assert s.push({}) == {} and s.push({"a": torch.zeros(0, dtype=torch.int16, device="cuda")})["a"].numel() == 0
        assert _lib.launch_count() == c0
        s.close("a")
        got = [[] for _ in xs]
        pos = [0] * 3
        for r in range(max(len(q) for q in sched)):
            chunks = {k: torch.from_numpy(xs[k][pos[k]:pos[k] + sched[k][r]]).cuda() for k in range(3) if r < len(sched[k])}
            final = [k for k in chunks if r == len(sched[k]) - 1]
            for k in chunks:
                pos[k] += chunks[k].numel()
            c0 = _lib.launch_count()
            for k, v in s.push(chunks, final).items():
                got[k].append(v)
            assert _lib.launch_count() - c0 <= 2
        runs.append([torch.cat(g) for g in got])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


# ---- decode sessions and pools -------------------------------------------------------------------------------------
def _net(shape, bf16, seed):
    from oracle import wavenet_oracle as O
    from tests.util import our_model
    cfg = O.Config(*shape)
    net = our_model(cfg, O.make_params(cfg, seed)).eval()
    net.decode_math = "bf16" if bf16 else "fp32"
    return cfg, net


def _aux_case(rng, lengths, fs=16000, fftl=1024, hop=80):
    xs = _signals(rng, lengths, True)
    mean, scale = rng.randn(80) - 4, 0.5 + rng.rand(80)
    from pytorchwavenetvocoder_b200.utils.device_loader import _f32_scaler_mode
    mode = _f32_scaler_mode()
    feats = melspc_batch(xs, fs, fftl, hop, 80, highpass_cutoff=70)
    if mode == 0:
        h = [((f.astype(np.float64) - mean).astype(np.float32).astype(np.float64) / scale).astype(np.float32)
             for f in feats]
    else:
        h = [(f - mean.astype(np.float32)) / scale.astype(np.float32) for f in feats]
    H = np.zeros((len(xs), 80, max(len(f) for f in h)), dtype=np.float32)
    for b, f in enumerate(h):
        H[b, :, :len(f)] = f.T
    return xs, (mean, scale), torch.from_numpy(H).cuda(), [len(f) * hop - 1 for f in h]


@pytest.mark.parametrize("shape,bf16", [((256, 80, 64, 64, 4, 2, 2, 80), False), ((256, 80, 512, 256, 10, 3, 2, 80), True)])
def test_session_fed_by_stream_equals_one_shot(shape, bf16):
    cfg, net = _net(shape, bf16, 71)
    rng = np.random.RandomState(4)
    xs, scaler, H, n_list = _aux_case(rng, [3000, 4100, 1234])
    B = len(xs)
    X = torch.full((B, 1), 128, dtype=torch.long, device="cuda")
    with torch.no_grad():
        torch.manual_seed(5)
        want = net._decode(X, H, n_list, "sampling").cpu().numpy()
        torch.manual_seed(5)
        sess = net.decode_session(X, n_list)
        s = MelspcStream(16000, 1024, 80, 80, highpass_cutoff=70, scaler=scaler)
        got = [[] for _ in range(B)]
        bufs = [torch.zeros(80, 0, device="cuda") for _ in range(B)]
        ended, pos, T, fed = [False] * B, [0] * B, H.size(2), 0
        while not sess.done:
            live = [b for b in range(B) if not ended[b]]
            if live:
                chunks = {b: torch.from_numpy(xs[b][pos[b]:pos[b] + 700]).cuda() for b in live}
                final = [b for b in live if pos[b] + 700 >= len(xs[b])]
                for b, a in s.push(chunks, final).items():
                    bufs[b] = torch.cat([bufs[b], a], 1)
                    pos[b] += 700
                for b in final:
                    ended[b] = True
            k = min(T if ended[b] else fed + bufs[b].size(1) for b in range(B)) - fed
            if k <= 0:
                continue
            h = torch.zeros(B, 80, k, device="cuda")
            for b in range(B):
                n = min(k, bufs[b].size(1))
                h[b, :, :n] = bufs[b][:, :n]
                bufs[b] = bufs[b][:, n:]
            out = sess.step(h)
            for b, c in enumerate(sess.last_counts):
                got[b].append(out[b, :c].cpu().numpy())
            fed += k
    for b in range(B):
        assert np.array_equal(np.concatenate(got[b]), want[b, :n_list[b]]), b


def test_pool_fed_by_stream_equals_one_shot():
    cfg, net = _net((256, 80, 512, 256, 10, 3, 2, 80), True, 73)
    rng = np.random.RandomState(6)
    xs, scaler, H, n_list = _aux_case(rng, [2500, 3300, 900, 4000])
    B = len(xs)
    X = torch.full((B, 1), 128, dtype=torch.long, device="cuda")
    with torch.no_grad():
        want = net._decode(X, H, n_list, "sampling", seed=1234, kernel="bf16").cpu().numpy()
        pool = net.decode_pool(4, "sampling", 1234)
        s = MelspcStream(16000, 1024, 80, 80, highpass_cutoff=70, scaler=scaler)
        for k in range(B):
            pool.admit(X[k], n_list[k], stream=k)
        got = {k: [] for k in range(B)}
        pos = [0] * B
        while not all(pool.finished(k) for k in range(B)):
            chunks = {k: torch.from_numpy(xs[k][pos[k]:pos[k] + 500]).cuda() for k in range(B) if pos[k] < len(xs[k])}
            final = [k for k in chunks if pos[k] + 500 >= len(xs[k])]
            for k, a in s.push(chunks, final).items():
                pos[k] += 500
                if a.size(1):
                    pool.feed(k, a)
            for k, c in pool.step().items():
                got[k].append(c.cpu().numpy())
    for k in range(B):
        assert np.array_equal(np.concatenate(got[k]), want[k, :n_list[k]]), k


# ---- bin/resynthesize.py -------------------------------------------------------------------------------------------
def _cli(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", module] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=900)
    assert r.returncode == 0, r.stdout.decode()[-3000:]


def test_cli_equals_feature_extract_then_decode(tmp_path):
    from oracle import mlsa_oracle as M
    from pytorchwavenetvocoder_b200.nets import WaveNet
    from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav_int16
    U, D_ = 80, 80
    rng = np.random.RandomState(12)
    torch.manual_seed(0)
    net = WaveNet(256, D_, 64, 64, 3, 2, 2, U)
    expdir, wavdir = tmp_path / "exp", tmp_path / "wav"
    expdir.mkdir()
    wavdir.mkdir()
    torch.save({"model": net.state_dict()}, str(expdir / "checkpoint-final.pkl"))
    conf = argparse.Namespace(n_quantize=256, n_aux=D_, n_resch=64, n_skipch=64, dilation_depth=3, dilation_repeat=2,
                              kernel_size=2, upsampling_factor=U, use_upsampling_layer=True, feature_type="melspc",
                              use_speaker_code=False)
    torch.save(conf, str(expdir / "model.conf"))
    for i, n in enumerate([1500, 2400, 1999, 800]):
        write_wav_int16(str(wavdir / ("r%d.wav" % i)), 16000, _signals(rng, [n], True)[0])
    stats = str(tmp_path / "stats.npz")
    write_hdf5(stats, "/melspc/mean", rng.randn(D_) - 4)
    write_hdf5(stats, "/melspc/scale", 0.5 + rng.rand(D_))
    write_hdf5(stats, "/mlsa/coef", M.convert_mcep_to_mlsa_coef(rng.randn(25) * 0.5, 0.5, 0.41))
    write_hdf5(stats, "/mlsa/alpha", 0.41)
    hdf5dir = str(tmp_path / "feats")
    _cli("pytorchwavenetvocoder_b200.bin.feature_extract", ["--waveforms", str(wavdir), "--hdf5dir", hdf5dir,
                                                            "--feature_type", "melspc", "--save_wav", "false",
                                                            "--fmin", "", "--fmax", ""])
    ck = str(expdir / "checkpoint-final.pkl")
    for bs in ("3", "1"):
        for ns in ([], ["--noise_shaping"]):
            common = ["--checkpoint", ck, "--stats", stats, "--fs", "16000", "--batch_size", bs, "--seed", "3"] + ns
            ref = str(tmp_path / ("dec_%s_%d" % (bs, len(ns))))
            _cli("pytorchwavenetvocoder_b200.bin.decode", common + ["--feats", hdf5dir, "--outdir", ref])
            for chunk in ("0", "80", "1000"):
                od = str(tmp_path / ("res_%s_%d_%s" % (bs, len(ns), chunk)))
                _cli("pytorchwavenetvocoder_b200.bin.resynthesize", common + ["--waveforms", str(wavdir), "--outdir", od,
                                                                              "--chunk_samples", chunk, "--fmin", ""])
                for i in range(4):
                    want = open(os.path.join(ref, "r%d.wav" % i), "rb").read()
                    got = open(os.path.join(od, "r%d.wav" % i), "rb").read()
                    assert len(want) > 44 and got == want, (bs, ns, chunk, i)
