# -*- coding: utf-8 -*-
"""GPU tier of held-out scoring: WaveNet.score and wnb_cross_entropy_rows against the float64 oracle, batch-composition
invariance, determinism, windowed against whole-utterance scoring, forward_loss, the pinned launch list,
bin/evaluate.py and train.py --dev_interval."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.score_reference import rows_ce
from tests.util import our_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SMALL_UP = O.Config(256, 28, 16, 32, 4, 2, 2, 4)          # ks 2, up-sampling layer
SMALL_KS3 = O.Config(256, 28, 16, 32, 4, 2, 3, 0)         # ks 3, aux at the sample rate
SPEAKER = O.Config(256, 31, 16, 32, 3, 2, 2, 0)           # 28 features + a 3-column speaker code, no up-sampling
BASE = O.Config(256, 28, 64, 512, 10, 3, 2, 80)           # the BASELINE shape
SHALLOW = O.Config(256, 28, 64, 512, 10, 1, 2, 80)        # 64/512, rf 1024


def _utts(cfg, lengths, seed):
    """[(x_in, t, h)] of random codes and features, T a multiple of U (as utterance_arrays gives)."""
    rng = np.random.RandomState(seed)
    U = cfg.upsampling_factor
    out = []
    for T in lengths:
        codes = rng.randint(0, 256, size=T + 1).astype(np.int64)
        h = rng.standard_normal((cfg.n_aux, T // U if U > 0 else T)).astype(np.float32)
        out.append((codes[:T], codes[1:], h))
    return out


def _batch(cfg, utts, T):
    from pytorchwavenetvocoder_b200.utils.scoring import _upload
    return _upload(utts, T, cfg.upsampling_factor, cfg.n_aux)


def _oracle_rows(cfg, p, utts, start):
    """float64 (nll, count) per utterance from the oracle's logits, each utterance alone (tests/score_reference.py)."""
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    nll, cnt = [], []
    for x, t, h in utts:
        if len(x) <= start:
            nll.append(0.0)
            cnt.append(0)
            continue
        lg = O.forward(cfg, p64, x[None], h[None].astype(np.float64))
        n, c = rows_ce(lg, t[None], [len(x)], start)
        nll.append(n[0])
        cnt.append(c[0])
    return np.array(nll), np.array(cnt)


def _round(cfg, T):
    U = cfg.upsampling_factor
    return T // U * U if U > 0 else T


@pytest.mark.parametrize("name,cfg,mode,start", [
    ("ks2_up", SMALL_UP, "fp32", None), ("ks2_up_from0", SMALL_UP, "fp32", 0), ("ks3_u0", SMALL_KS3, "fp32", None),
    ("speaker", SPEAKER, "fp32", None), ("base", BASE, "fp32", None), ("base", BASE, "tf32", None),
    ("base", BASE, "bf16", None)])
def test_score_matches_float64_oracle(name, cfg, mode, start):
    p = O.make_params(cfg, 11)
    net = our_model(cfg, p, math_mode=mode)
    rf = cfg.receptive_field
    lengths = [_round(cfg, rf + 700), _round(cfg, rf + 333), cfg.upsampling_factor or rf + 1]
    utts = _utts(cfg, lengths, 3)
    xb, tb, hb = _batch(cfg, utts, max(lengths))
    nll, cnt = net.score(xb, hb, tb, lengths, start)
    nll, cnt = nll.cpu().numpy(), cnt.cpu().numpy()
    s0 = rf if start is None else start
    want, wcnt = _oracle_rows(cfg, p, utts, s0)
    assert np.array_equal(cnt, wcnt), (cnt, wcnt)
    live = wcnt > 0
    assert not np.isnan(nll).any() and (nll[~live] == 0).all()
    if mode == "fp32":
        rel = np.abs(nll[live] - want[live]) / np.abs(want[live])
        print("%s %s: worst relative error of the summed NLL %.2e" % (name, mode, rel.max()))
        assert rel.max() <= 1e-5
    else:   # DESIGN.md section 4: the loss bound of each mode, per sample
        err = np.abs(nll[live] / cnt[live] - want[live] / wcnt[live])
        print("%s %s: worst error of nats / sample %.2e" % (name, mode, err.max()))
        assert err.max() <= {"tf32": 2.5e-3, "bf16": 1.2e-3}[mode]


@pytest.mark.parametrize("cfg,mode", [(SMALL_UP, "fp32"), (SMALL_KS3, "fp32"), (SHALLOW, "tf32"), (SHALLOW, "bf16")])
def test_batch_composition_and_runs_bit_identical(cfg, mode):
    net = our_model(cfg, O.make_params(cfg, 5), math_mode=mode)
    rf = cfg.receptive_field
    U = max(cfg.upsampling_factor, 1)
    lengths = [_round(cfg, rf + 900), _round(cfg, rf + 1) or U, _round(cfg, rf + 413), U]   # two shorter than rf + 2
    utts = _utts(cfg, lengths, 9)
    alone = []
    for u, T in zip(utts, lengths):
        xb, tb, hb = _batch(cfg, [u], T)
        alone.append(net.score(xb, hb, tb, [T]))
    for order, pad in (([0, 1, 2, 3], 0), ([3, 2, 1, 0], 5 * U), ([2, 0], 17 * U)):
        us = [utts[i] for i in order]
        T = max(lengths[i] for i in order) + pad
        xb, tb, hb = _batch(cfg, us, T)
        for run in range(2):
            nll, cnt = net.score(xb, hb, tb, [lengths[i] for i in order])
            for r, i in enumerate(order):
                assert torch.equal(nll[r], alone[i][0][0]) and torch.equal(cnt[r], alone[i][1][0]), (mode, order, r)
    assert int(alone[3][1][0]) == 0 and float(alone[3][0][0]) == 0.0


@pytest.mark.parametrize("cfg,mode", [(SMALL_UP, "fp32"), (SMALL_KS3, "fp32"), (SHALLOW, "fp32"), (SHALLOW, "tf32"),
                                      (SHALLOW, "bf16")])
def test_windowed_scoring_equals_whole(cfg, mode):
    from pytorchwavenetvocoder_b200.utils.scoring import score_windows, window_unit
    net = our_model(cfg, O.make_params(cfg, 6), math_mode=mode)
    rf = cfg.receptive_field
    unit = window_unit(cfg.upsampling_factor)
    lengths = sorted([_round(cfg, 3 * rf + 5 * unit + 7), _round(cfg, 2 * rf + 11), _round(cfg, rf + 3 * unit)],
                     reverse=True)
    utts = _utts(cfg, lengths, 4)
    xb, tb, hb = _batch(cfg, utts, lengths[0])
    for start in (rf, 0, rf + unit + 5):
        whole = net.score(xb, hb, tb, lengths, start)
        for L in (unit, 3 * unit):
            out = (torch.zeros(3, dtype=torch.float64, device="cuda"), torch.zeros(3, dtype=torch.int64, device="cuda"))
            score_windows(net, utts, L, start, out)
            assert torch.equal(out[1], whole[1]), (start, L)
            assert torch.equal(out[0], whole[0]), (mode, start, L, out[0] - whole[0])


@pytest.mark.parametrize("cfg,mode", [(SMALL_UP, "fp32"), (SHALLOW, "tf32"), (SHALLOW, "bf16")])
def test_score_equals_forward_loss_on_one_window(cfg, mode):
    net = our_model(cfg, O.make_params(cfg, 8), math_mode=mode)
    rf = cfg.receptive_field
    T = _round(cfg, rf + 640)
    utts = _utts(cfg, [T, T], 2)
    xb, tb, hb = _batch(cfg, utts, T)
    nll, cnt = net.score(xb, hb, tb, [T, T])
    with torch.no_grad():
        loss = net.forward_loss(xb, hb, tb, rf)
    got = float(nll.sum()) / int(cnt.sum())
    assert int(cnt.sum()) == 2 * (T - rf)
    assert abs(got - float(loss)) <= 2e-6 * abs(got), (got, float(loss))


@pytest.mark.parametrize("Q", [256, 100])
def test_position_value_is_wnb_cross_entropy(Q):
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(Q)
    B = 37
    logits = torch.randn(B, 1, Q, device="cuda", generator=g) * 4
    target = torch.randint(0, Q, (B, 1), device="cuda", generator=g)
    nll = torch.zeros(B, dtype=torch.float64, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int64, device="cuda")
    lengths = torch.ones(B, dtype=torch.int64, device="cuda")
    st = _lib.stream()
    _lib.check(lib.wnb_cross_entropy_rows(logits.data_ptr(), target.data_ptr(), lengths.data_ptr(), 0, nll.data_ptr(),
                                          cnt.data_ptr(), B, 1, Q, st), "rows")
    for b in range(B):
        one = torch.zeros(1, dtype=torch.float64, device="cuda")
        _lib.check(lib.wnb_cross_entropy(logits[b].data_ptr(), target[b].data_ptr(), one.data_ptr(), None, 1, 1, Q, 0,
                                         st), "ce")
        assert torch.equal(one[0], nll[b]), (Q, b)
    assert (cnt == 1).all()
    # a target out of range gives NaN, as wnb_cross_entropy flags it
    target[0, 0] = Q
    nll.zero_()
    _lib.check(lib.wnb_cross_entropy_rows(logits.data_ptr(), target.data_ptr(), lengths.data_ptr(), 0, nll.data_ptr(),
                                          None, B, 1, Q, st), "rows")
    assert torch.isnan(nll[0]) and not torch.isnan(nll[1:]).any()


def _kernels(fn, tries=3):
    """(library launches, sorted names of this library's kernels, sorted names of every other kernel) of ``fn()``.

    The library counts its own launches; the profiler's kernel records are the names.  The profiler can lose a kernel
    record now and then, so a capture with fewer library kernel records than library launches is taken again (``fn``
    has no side effects that change its launches), up to ``tries`` times.  A shortfall that repeats is returned as it
    is and fails the caller's count; so does any surplus, which no retry hides."""
    from pytorchwavenetvocoder_b200 import _lib
    for attempt in range(tries):
        torch.cuda.synchronize()
        l0 = _lib.launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        launches = _lib.launch_count() - l0
        ks = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
              and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
        lib = sorted(n for n in ks if "wnb::" in n)
        if len(lib) >= launches:
            break
        print("capture %d: %d library kernel records for %d library launches; capturing again"
              % (attempt, len(lib), launches))
    return launches, lib, sorted(n for n in ks if "wnb::" not in n)


@pytest.mark.parametrize("mode", ["tf32", "fp32", "bf16"])
def test_launch_list_is_pinned(mode):
    """At the BASELINE shape, score launches the no-grad forward's kernels plus one wnb_cross_entropy_rows.  Under tf32
    every kernel is this library's.  Under fp32 and bf16 the forward packs the weights with torch ops on every call
    (the only torch kernels), and score runs exactly those packing kernels, no other."""
    net = our_model(BASE, O.make_params(BASE, 1), math_mode=mode)
    T = _round(BASE, BASE.receptive_field + 4000)
    utts = _utts(BASE, [T, T - 800], 1)
    xb, tb, hb = _batch(BASE, utts, T)
    lengths = torch.tensor([T, T - 800], dtype=torch.int64, device="cuda")
    net.score(xb, hb, tb, lengths)

    def fwd():
        with torch.no_grad():
            net(xb, hb)
    f_launch, f_lib, f_torch = _kernels(fwd)
    launches, lib, other = _kernels(lambda: net.score(xb, hb, tb, lengths))
    print("%s score launches: %d (forward %d); torch kernels %d: %s" % (mode, launches, f_launch, len(other),
                                                                      sorted(set(lib))))
    assert launches == f_launch + 1 and len(lib) == launches and len(f_lib) == f_launch
    assert sorted(lib) == sorted(f_lib + [n for n in lib if "cross_entropy_rows_kernel" in n])
    assert sum("cross_entropy_rows_kernel" in n for n in lib) == 1
    assert other == f_torch
    if mode == "tf32":
        assert other == [], other


def test_score_ping_pongs_the_activations():
    """tf32 at the BASELINE shape (the deferred-skip stack): score, and forward under no_grad, keep two residual
    buffers, not one per layer.  The peak is what two buffers, Z_all, skip, r1, logits and aux take."""
    net = our_model(BASE, O.make_params(BASE, 2), math_mode="tf32")
    B, T = 2, _round(BASE, BASE.receptive_field + 40000)
    utts = _utts(BASE, [T, T], 3)
    xb, tb, hb = _batch(BASE, utts, T)
    lengths = torch.tensor([T, T], dtype=torch.int64, device="cuda")
    L, R, S, Q, Ap = len(BASE.dilations), BASE.n_resch, BASE.n_skipch, BASE.n_quantize, 32
    two = 4 * B * T * (L * R + 2 * R + 2 * S + Q + Ap)
    every = 4 * B * T * (L * R + L * R + 2 * S + Q + Ap)
    net.score(xb, hb, tb, lengths)
    for fn in (lambda: net.score(xb, hb, tb, lengths), lambda: torch.no_grad()(net.forward)(xb, hb)):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        print("peak %.0f MB; two buffers %.0f MB, one per layer %.0f MB" % (peak / 2 ** 20, two / 2 ** 20,
                                                                           every / 2 ** 20))
        assert peak <= 1.02 * two + (8 << 20) and peak < 0.8 * every


def _corpus(tmp_path, cfg, n_frames, seed, stats_key="world"):
    from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav
    rng = np.random.RandomState(seed)
    U, D = cfg.upsampling_factor, cfg.n_aux
    d = tmp_path / ("c%d" % seed)
    d.mkdir()
    wavs, feats = [], []
    for i, nf in enumerate(n_frames):
        w, f = str(d / ("u%d.wav" % i)), str(d / ("u%d.npz" % i))
        write_wav(w, 0.4 * np.sin(np.arange(nf * U + 3) / (5.0 + i)) + 0.05 * rng.standard_normal(nf * U + 3), 16000)
        write_hdf5(f, "/world", rng.standard_normal((nf, D)))
        wavs.append(w)
        feats.append(f)
    wl, fl, stats = str(d / "wav.scp"), str(d / "feats.scp"), str(d / "stats.npz")
    open(wl, "w").write("\n".join(wavs) + "\n")
    open(fl, "w").write("\n".join(feats) + "\n")
    write_hdf5(stats, "/" + stats_key + "/mean", np.zeros(D))
    write_hdf5(stats, "/" + stats_key + "/scale", np.ones(D))
    return wavs, feats, wl, fl, stats


def test_evaluate_writes_what_the_api_returns(tmp_path):
    import argparse
    from pytorchwavenetvocoder_b200.bin import evaluate as E
    from pytorchwavenetvocoder_b200.bin.decode import load_scaler
    from pytorchwavenetvocoder_b200.utils.scoring import corpus_mean, load_utterance, score_utterances
    cfg = SMALL_UP
    wavs, feats, wl, fl, stats = _corpus(tmp_path, cfg, [60, 7, 75, 2, 40], 0)
    conf = argparse.Namespace(n_quantize=256, n_aux=28, n_resch=16, n_skipch=32, dilation_depth=4, dilation_repeat=2,
                              kernel_size=2, upsampling_factor=4, use_upsampling_layer=True, use_speaker_code=False,
                              feature_type="world", math_mode="fp32")
    confp = str(tmp_path / "model.conf")
    torch.save(conf, confp)
    ckpts = []
    for s in (1, 2):
        net = our_model(cfg, O.make_params(cfg, s))
        ckpts.append(str(tmp_path / ("checkpoint-%d.pkl" % s)))
        torch.save({"model": net.state_dict()}, ckpts[-1])
    out = str(tmp_path / "scores.tsv")
    # a budget below the longest utterance: it is scored in windows
    E.main(["--waveforms", wl, "--feats", fl, "--checkpoint"] + ckpts +
           ["--stats", stats, "--config", confp, "--outfile", out, "--batch_samples", "200"])
    rows = [l.rstrip("\n").split("\t") for l in open(out)][1:]
    assert len(rows) == 2 * (len(wavs) + 1)
    scaler = load_scaler(stats, "world")
    utts = [load_utterance(w, f, conf, scaler) for w, f in zip(wavs, feats)]
    for c, ck in enumerate(ckpts):
        net = E.build_model(conf, ck, "fp32")
        nll, cnt = score_utterances(net, utts, 1 << 20)
        mine = rows[c * (len(wavs) + 1):(c + 1) * (len(wavs) + 1)]
        assert [r[1] for r in mine] == ["u%d" % i for i in range(len(wavs))] + ["<corpus>"]
        for r, v, n in zip(mine, nll, cnt):
            assert r[0] == ck and int(r[2]) == n and float(r[3]) == v, (r, v, n)
        s, n, mean = corpus_mean(nll, cnt)
        assert float(mine[-1][3]) == s and int(mine[-1][2]) == n and float(mine[-1][4]) == mean
    assert cnt[3] == 0 and cnt[1] == 0                     # shorter than the receptive field: nothing scored


def _train(tmp_path, tag, extra, math_mode, n_gpus=1):
    """Train the SMALL_UP shape for 7 steps on corpus c0, with ``extra`` flags and corpus c1 as the held-out list."""
    c0 = tmp_path / "c0"
    wl, fl, stats = str(c0 / "wav.scp"), str(c0 / "feats.scp"), str(c0 / "stats.npz")
    dev = ["--dev_waveforms", str(tmp_path / "c1" / "wav.scp"), "--dev_feats", str(tmp_path / "c1" / "feats.scp")]
    expdir = str(tmp_path / tag)
    args = ["--waveforms", wl, "--feats", fl, "--stats", stats, "--expdir", expdir, "--n_resch", "16", "--n_skipch",
            "32", "--dilation_depth", "4", "--dilation_repeat", "2", "--upsampling_factor", "4", "--batch_length", "160",
            "--batch_size", "2", "--intervals", "2", "--checkpoint_interval", "3", "--iters", "7", "--math_mode",
            math_mode, "--n_gpus", str(n_gpus), "--verbose", "1"] + (dev + extra if extra else [])
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.train"] + args, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    log = r.stdout.decode()
    assert r.returncode == 0, log[-3000:]
    return expdir, log


@pytest.mark.parametrize("math_mode,n_gpus", [("fp32", 1), ("tf32", 1), ("tf32", 2)])
def test_train_dev_loss_leaves_checkpoints_unchanged(tmp_path, math_mode, n_gpus):
    if torch.cuda.device_count() < n_gpus:
        pytest.skip("needs %d GPUs" % n_gpus)
    _corpus(tmp_path, SMALL_UP, [60, 75, 50], 0)
    _corpus(tmp_path, SMALL_UP, [40, 33, 8, 51, 20], 1)
    base, log0 = _train(tmp_path, "plain", None, math_mode, n_gpus)
    dev, log1 = _train(tmp_path, "dev", ["--dev_interval", "2"], math_mode, n_gpus)
    assert "dev loss" not in log0
    lines = [l for l in log1.splitlines() if "dev loss" in l]
    assert [l.split("(iter:")[1].split(")")[0] for l in lines] == ["2", "4", "6", "7"], lines
    for name in ("checkpoint-3.pkl", "checkpoint-6.pkl", "checkpoint-final.pkl"):
        a = torch.load(os.path.join(base, name), map_location="cpu", weights_only=False)
        b = torch.load(os.path.join(dev, name), map_location="cpu", weights_only=False)
        for k in a["model"]:
            assert torch.equal(a["model"][k], b["model"][k]), (name, k)
        with open(os.path.join(base, name), "rb") as fa, open(os.path.join(dev, name), "rb") as fb:
            assert fa.read() == fb.read(), name
    # the logged figure is the API's corpus mean of the final model on the same list
    from pytorchwavenetvocoder_b200.bin.decode import load_scaler
    from pytorchwavenetvocoder_b200.bin.evaluate import build_model, file_lists
    from pytorchwavenetvocoder_b200.utils.scoring import corpus_mean, load_utterance, score_utterances
    conf = torch.load(os.path.join(dev, "model.conf"), weights_only=False)
    net = build_model(conf, os.path.join(dev, "checkpoint-final.pkl"), math_mode)
    wl, fl = file_lists(str(tmp_path / "c1" / "wav.scp"), str(tmp_path / "c1" / "feats.scp"))
    scaler = load_scaler(conf.stats, "world")
    utts = [load_utterance(w, f, conf, scaler) for w, f in zip(wl, fl)]
    mean = corpus_mean(*score_utterances(net, utts, 1 << 21))[2]
    assert lines[-1].split("dev loss = ")[1].split(" ")[0] == "%.6f" % mean
