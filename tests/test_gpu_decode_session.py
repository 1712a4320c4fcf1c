# -*- coding: utf-8 -*-
"""GPU tier: resumable decode sessions (``WaveNet.decode_session``, the ``_at`` decode entry points).

Chunked decoding must equal one-shot decoding BIT FOR BIT -- the codes and the teacher-check logits -- in argmax mode,
with supplied uniforms and with in-kernel Philox, on every launch form:
* all eight ``decode_warp_kernel`` forms (reached as in test_gpu_decode_forms.py and asserted through
  ``wnb_decode_warp_form``), the speaker-code shape (U = 0, A = 31), stream and direct with 1, 2 and 4 utterances per CTA,
  and the bf16 decoder at 512/256 (B = 3) and 256/256 (B = 70: two clusters);
* chunk schedules of 1 frame, of random sizes, with boundaries at a wrap of the largest dilation ring, and (seed longer
  than the receptive field) a first chunk inside the warm-up; ragged lengths finish in different chunks;
* 10 000 Philox steps at the bench shape in 80-sample chunks;
* two sessions interleaved on one model, and on two streams, equal each run alone;
* the library launches of one one-shot decode (a one-call session) on each kernel, the count bench.py reports;
* every error case, and ``bin/decode.py --chunk_frames 7`` writing the same wav bytes as the one-shot run."""
import argparse
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHALLOW = (256, 28, 64, 512, 4, 2, 2, 4)      # L = 8, largest dilation 8
BENCH = (256, 28, 64, 512, 10, 3, 2, 80)      # the bench's decode shape
_MODELS = {}


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _model(t, decode_math="fp32"):
    key = (t, decode_math)
    if key not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 31 + len(_MODELS))).eval()
        net.decode_math = decode_math
        _MODELS[key] = (cfg, net)
    return _MODELS[key]


def _warp_form(B, L):
    from pytorchwavenetvocoder_b200 import _lib
    f = (ctypes.c_int32 * 4)()
    _lib.check(_lib.load().wnb_decode_warp_form(B, L, f), "decode_warp_form")
    return tuple(int(v) for v in f)


def _inputs(cfg, B, T0, max_n, seed):
    rng = np.random.RandomState(seed)
    U = max(cfg.upsampling_factor, 1)
    x = torch.from_numpy(rng.randint(0, cfg.n_quantize, size=(B, T0))).cuda()
    h = torch.from_numpy(rng.standard_normal((B, cfg.n_aux, (T0 + max_n + U - 1) // U + 1)).astype(np.float32)).cuda()
    n_list = [int(v) for v in rng.randint(1, max_n + 1, size=B)]
    n_list[0] = 1
    if B > 1:
        n_list[1] = max_n
    return x, h, n_list


def _schedule(kind, cfg, T0, nf, seed):
    """chunk sizes in frames (covering nf frames)"""
    U = max(cfg.upsampling_factor, 1)
    P = max(T0, cfg.receptive_field)
    n_pad, dmax = P - T0, max(cfg.dilations)
    if kind == "ones":
        return [1] * nf
    if kind == "random":   # small enough that the frames after the warm-up still take several calls
        rng = np.random.RandomState(seed)
        after = nf - (P - 1 - n_pad) // U - 1
        return [int(v) for v in rng.randint(1, max(2, min(7, after // 3)), size=nf)]
    assert kind == "wrap"   # every call after the first starts at a multiple of the largest dilation (when one fits)
    step = dmax // math.gcd(U, dmax)
    first = [f for f in range(1, nf - step) if (n_pad + f * U) % dmax == 0 and n_pad + f * U >= P]
    return [first[0]] + [step] * nf if first else [1] * nf


def _short_seed(cfg):
    """a seed shorter than the receptive field with n_pad a multiple of the largest dilation"""
    return 1 + (cfg.receptive_field - 1) % max(cfg.dilations)


def _chunked(net, x, h, n_list, mode, sched, uniforms=None, seed=None, kernel="auto"):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    with torch.no_grad():
        s = DecodeSession(net, x, n_list, mode, seed, uniforms, True, kernel)
        B, Q = len(n_list), net.n_quantize
        codes = [[] for _ in range(B)]
        logits = [[] for _ in range(B)]
        f0 = 0
        calls = 0
        for F in sched:
            if s.done:
                break
            gen, lg = s.step(h[:, :, f0:f0 + F])
            f0 += F
            calls += int(gen.size(1) > 0)
            gen, lg = gen.cpu().numpy(), lg.cpu().numpy()
            for b, c in enumerate(s.last_counts):
                codes[b].append(gen[b, :c])
                logits[b].append(lg[b, :c])
        assert s.done, "schedule too short"
    return ([np.concatenate(c) for c in codes], [np.concatenate(l).reshape(-1, Q) for l in logits], s.kernel, calls)


def _oneshot(net, x, h, n_list, mode, uniforms=None, seed=None, kernel="auto"):
    with torch.no_grad():
        gen, lg = net._decode(x, h, n_list, mode, uniforms=uniforms, return_logits=True, seed=seed, kernel=kernel)
    return gen.cpu().numpy(), lg.cpu().numpy(), net.last_decode_kernel


def _check_modes(net, cfg, x, h, n_list, kernel, seed, scheds):
    """argmax / supplied uniforms / Philox, each with its schedule: chunked == one-shot, codes and logits, bit for bit"""
    B, max_n = len(n_list), max(n_list)
    uni = torch.from_numpy(np.random.RandomState(seed).uniform(size=(B, max_n)).astype(np.float32))
    runs = {"argmax": ("argmax", None, None), "uniforms": ("sampling", uni, None), "philox": ("sampling", None, seed)}
    for (name, (mode, u, sd)), sched in zip(runs.items(), scheds):
        gen, lg, k1 = _oneshot(net, x, h, n_list, mode, u, sd, kernel)
        codes, logits, k2, calls = _chunked(net, x, h, n_list, mode, sched, u, sd, kernel)
        assert k1 == k2, (name, k1, k2)
        assert calls > 1, (name, sched)
        for b in range(B):
            assert np.array_equal(codes[b], gen[b, :n_list[b]]), (name, b)
            assert np.array_equal(logits[b].view(np.uint32), lg[b, :n_list[b]].view(np.uint32)), (name, b)
    return k1


WARP_FORMS = {
    "1x16_big_cl2": (BENCH, lambda n: n // 2 - 1, None, (1, 16, 2, 1)),
    "1x16_big_cl1": (BENCH, lambda n: n // 2 + 3, None, (1, 16, 1, 1)),
    "1x16_small_cl2": (SHALLOW, lambda n: n // 2 - 1, "0", (1, 16, 2, 0)),
    "1x16_small_cl1": (SHALLOW, lambda n: n - 1, "0", (1, 16, 1, 0)),
    "2x16_big": (SHALLOW, lambda n: n + 7, None, (2, 16, 1, 1)),
    "2x16_small": (SHALLOW, lambda n: 2 * n - 1, "0", (2, 16, 1, 0)),
    "4x8_big": ((256, 28, 64, 512, 3, 3, 2, 4), lambda n: 2 * n + 7, None, (4, 8, 1, 1)),
    "4x8_small": ((256, 28, 64, 512, 6, 2, 2, 4), lambda n: 2 * n + 9, "0", (4, 8, 1, 0)),
    "speaker_A31_U0": ((256, 31, 64, 512, 4, 2, 2, 0), lambda n: 5, None, (1, 16, 2, 1)),
}


@pytest.mark.parametrize("form_id", list(WARP_FORMS))
def test_warp_forms_chunked_equal_oneshot(form_id, monkeypatch):
    t, bfn, big, want = WARP_FORMS[form_id]
    if big is not None:
        monkeypatch.setenv("WNB_DECODE_BIG", big)
    cfg, net = _model(t)
    B = bfn(_nsm())
    assert _warp_form(B, len(cfg.dilations)) == want
    ci = list(WARP_FORMS).index(form_id)
    T0 = _short_seed(cfg) if ci % 2 == 0 else cfg.receptive_field + 9      # odd forms: a first chunk inside the warm-up
    max_n = 200 if cfg.upsampling_factor == 80 else 48
    x, h, n_list = _inputs(cfg, B, T0, max_n, 100 + ci)
    nf = h.size(2)
    scheds = [_schedule(k, cfg, T0, nf, ci) for k in ("ones", "random", "wrap")]
    assert _check_modes(net, cfg, x, h, n_list, "warp", 1000 + ci, scheds) == "warp"


@pytest.mark.parametrize("kernel", ["stream", "direct"])
@pytest.mark.parametrize("nu", [1, 2, 4])
def test_stream_direct_chunked_equal_oneshot(kernel, nu):
    cfg, net = _model(SHALLOW)
    nsm = _nsm()
    B = {1: 5, 2: nsm + 5, 4: 2 * nsm + 5}[nu]
    T0 = _short_seed(cfg) if nu != 2 else cfg.receptive_field + 9
    x, h, n_list = _inputs(cfg, B, T0, 40, 200 + nu)
    scheds = [_schedule(k, cfg, T0, h.size(2), nu) for k in ("wrap", "ones", "random")]
    assert _check_modes(net, cfg, x, h, n_list, kernel, 2000 + nu, scheds) == kernel


BF16 = {"arctic_512_256_B3": ((256, 28, 512, 256, 10, 3, 2, 80), 3, 170),
        "256_256_B70": ((256, 28, 256, 256, 4, 2, 2, 4), 70, 40)}


@pytest.mark.parametrize("case", list(BF16))
def test_bf16_chunked_equal_oneshot(case):
    t, B, max_n = BF16[case]
    cfg, net = _model(t, "bf16")
    x, h, n_list = _inputs(cfg, B, 1, max_n, 300)
    scheds = [_schedule(k, cfg, 1, h.size(2), 3) for k in ("random", "ones", "wrap")]
    assert _check_modes(net, cfg, x, h, n_list, "auto", 3000, scheds) == "bf16"


def test_long_philox_run_in_80_sample_chunks():
    cfg, net = _model(BENCH)
    B, n = 4, 10000
    x, h, _ = _inputs(cfg, B, 1, n, 400)
    n_list = [n, n - 37, n - 80, 5000]
    gen, lg, k1 = _oneshot(net, x, h, n_list, "sampling", seed=1234)
    codes, logits, k2, calls = _chunked(net, x, h, n_list, "sampling", [1] * h.size(2), seed=1234)
    assert k1 == k2 == "warp" and calls >= n // 80
    for b in range(B):
        assert np.array_equal(codes[b], gen[b, :n_list[b]]), b
        assert np.array_equal(logits[b].view(np.uint32), lg[b, :n_list[b]].view(np.uint32)), b


# library launches of one _decode call: the decode launch, after the parallel warm-up on warp (the front conv and one
# launch per layer but the last: L = 30 here) and on bf16 (the front conv, then a gate and a res launch per layer but the
# last: L = 8 here).  bench.py reports this count as gpu_launches.
LAUNCHES = {
    "warp_cl2": (WARP_FORMS["1x16_big_cl2"], "auto", "warp", 31),
    "warp_cl1": (WARP_FORMS["1x16_big_cl1"], "auto", "warp", 31),
    "stream": ((SHALLOW, lambda n: 5, None, None), "stream", "stream", 1),
    "direct": ((SHALLOW, lambda n: 5, None, None), "direct", "direct", 1),
    "bf16": (((256, 28, 256, 256, 4, 2, 2, 4), lambda n: 3, None, None), "auto", "bf16", 16),
}


@pytest.mark.parametrize("case", list(LAUNCHES))
def test_oneshot_launch_count(case):
    from pytorchwavenetvocoder_b200 import _lib
    (t, bfn, _, form), kernel, ran, want = LAUNCHES[case]
    cfg, net = _model(t, "bf16" if ran == "bf16" else "fp32")
    B = bfn(_nsm())
    if form is not None:
        assert _warp_form(B, len(cfg.dilations)) == form
    x, h, n_list = _inputs(cfg, B, 1, 8, 900)
    l0 = _lib.launch_count()
    net._decode(x, h, n_list, "sampling", seed=3, kernel=kernel)
    launches = _lib.launch_count() - l0
    assert net.last_decode_kernel == ran
    assert launches == want, (case, launches)


def test_sessions_are_isolated():
    """two sessions on one model, interleaved call by call on one stream and on two streams, equal each run alone"""
    cfg, net = _model(SHALLOW)
    xa, ha, na = _inputs(cfg, 3, 1, 40, 500)
    xb, hb, nb = _inputs(cfg, 5, 1, 40, 501)
    alone_a = net._decode(xa, ha, na, "sampling", seed=7).cpu().numpy()
    alone_b = net._decode(xb, hb, nb, "sampling", seed=8).cpu().numpy()
    for two_streams in (False, True):
        sa, sb = net.decode_session(xa, na, seed=7), net.decode_session(xb, nb, seed=8)
        streams = (torch.cuda.Stream(), torch.cuda.Stream()) if two_streams else (None, None)
        got = {"a": [[] for _ in na], "b": [[] for _ in nb]}
        f = 0
        while not (sa.done and sb.done):
            for key, s, hh, st in (("a", sa, ha, streams[0]), ("b", sb, hb, streams[1])):
                if s.done:
                    continue
                if st is not None:
                    st.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(st) if st is not None else torch.cuda.stream(torch.cuda.current_stream()):
                    out = s.step(hh[:, :, f:f + 2])
                    torch.cuda.current_stream().synchronize()
                    out = out.cpu().numpy()
                for i, c in enumerate(s.last_counts):
                    got[key][i].append(out[i, :c])
            f += 2
        for key, alone, nl in (("a", alone_a, na), ("b", alone_b, nb)):
            for i, n in enumerate(nl):
                assert np.array_equal(np.concatenate(got[key][i]), alone[i, :n]), (two_streams, key, i)


@pytest.mark.parametrize("kernel", ["warp", "stream", "direct", "bf16"])
def test_session_keeps_its_weight_snapshot(kernel):
    """in-place updates of the model between two calls (biases, a load_state_dict) do not reach a running session: it
    still equals the one-shot decode with the weights it was created with"""
    t = (256, 28, 256, 256, 4, 2, 2, 4) if kernel == "bf16" else SHALLOW
    cfg = O.Config(*t)
    net = our_model(cfg, O.make_params(cfg, 77)).eval()
    net.decode_math = "bf16" if kernel == "bf16" else "fp32"
    x, h, n_list = _inputs(cfg, 3, 1, 40, 800)
    k = "auto" if kernel == "bf16" else kernel
    want, _, _ = _oneshot(net, x, h, n_list, "sampling", seed=5, kernel=k)
    with torch.no_grad():
        s = _session_of(net, x, n_list, k)
        parts = [[] for _ in n_list]
        f = 0
        while not s.done:
            gen, _ = s.step(h[:, :, f:f + 3])
            for b, c in enumerate(s.last_counts):
                parts[b].append(gen.cpu().numpy()[b, :c])
            if f == 0:   # after the first call: change every bias in place, and the matrices through load_state_dict
                for name, prm in net.named_parameters():
                    if name.endswith("bias"):
                        prm.add_(0.5)
                sd = {kk: v + 0.01 for kk, v in net.state_dict().items()}
                net.load_state_dict(sd)
            f += 3
    changed, _, _ = _oneshot(net, x, h, n_list, "sampling", seed=5, kernel=k)
    assert not np.array_equal(changed[1, :n_list[1]], want[1, :n_list[1]])   # the update does change the output
    for b, n in enumerate(n_list):
        assert np.array_equal(np.concatenate(parts[b]), want[b, :n]), b


def _session_of(net, x, n_list, kernel):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    return DecodeSession(net, x, n_list, "sampling", 5, None, True, kernel)


def test_seed_follows_torch_manual_seed_and_pcm16():
    from pytorchwavenetvocoder_b200.nets import codes_to_pcm16
    cfg, net = _model(SHALLOW)
    x, h, n_list = _inputs(cfg, 3, 1, 30, 600)
    torch.manual_seed(99)
    gen = net._decode(x, h, n_list, "sampling")
    want = codes_to_pcm16(gen, 256).cpu().numpy()
    torch.manual_seed(99)
    s = net.decode_session(x, n_list)
    parts = [[] for _ in n_list]
    f = 0
    while not s.done:
        pcm = s.step_pcm16(h[:, :, f:f + 3])
        assert pcm.dtype == torch.int16
        pcm = pcm.cpu().numpy()
        for b, c in enumerate(s.last_counts):
            parts[b].append(pcm[b, :c])
        f += 3
    for b, n in enumerate(n_list):
        assert np.array_equal(np.concatenate(parts[b]), want[b, :n])


def test_session_errors():
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = _model(SHALLOW)
    x, h, n_list = _inputs(cfg, 3, 1, 8, 700)
    with pytest.raises(_lib.WnbError):                                  # CPU seed
        net.decode_session(x.cpu(), n_list)
    s = net.decode_session(x, n_list, mode="argmax")
    with pytest.raises(_lib.WnbError):                                  # CPU aux
        s.step(h.cpu())
    with pytest.raises(ValueError):                                     # wrong aux dimension
        s.step(h[:, :5])
    with pytest.raises(ValueError):                                     # another batch size
        s.step(h[:2])
    while not s.done:
        s.step(h[:, :, :4])
    with pytest.raises(RuntimeError):                                   # every utterance has finished
        s.step(h[:, :, :1])
    with pytest.raises(SystemExit):                                     # bad mode: like batch_fast_generate
        net.decode_session(x, n_list, mode="greedy")
    net.decode_math = "bf16"                                            # 64/512 is outside the bf16 decoder
    try:
        with pytest.raises(_lib.WnbError):
            net.decode_session(x, n_list)
    finally:
        net.decode_math = "fp32"
    with pytest.raises(ValueError):                                     # past 2^31 positions
        net.decode_session(x, [2 ** 31, 1, 1])


def _cli(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.decode"] + args, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    assert r.returncode == 0, r.stdout.decode()[-3000:]


@pytest.mark.parametrize("speaker", [False, True])
def test_cli_chunk_frames_writes_the_same_wavs(tmp_path, speaker):
    from pytorchwavenetvocoder_b200.nets import WaveNet
    from pytorchwavenetvocoder_b200.utils import write_hdf5
    U, D_, NS = 16, 28, 3
    n_aux = D_ + NS if speaker else D_
    rng = np.random.RandomState(4)
    torch.manual_seed(0)
    net = WaveNet(256, n_aux, 64, 128, 3, 2, 2, 0 if speaker else U)
    expdir, featdir = tmp_path / "exp", tmp_path / "feats"
    expdir.mkdir()
    featdir.mkdir()
    torch.save({"model": net.state_dict()}, str(expdir / "checkpoint-final.pkl"))
    conf = argparse.Namespace(n_quantize=256, n_aux=n_aux, n_resch=64, n_skipch=128, dilation_depth=3,
                              dilation_repeat=2, kernel_size=2, upsampling_factor=U, use_upsampling_layer=not speaker,
                              feature_type="world", use_speaker_code=speaker)
    torch.save(conf, str(expdir / "model.conf"))
    feats = []
    for i, nf in enumerate([20, 33, 27]):
        f = str(featdir / ("c%d.npz" % i))
        write_hdf5(f, "/world", rng.standard_normal((nf, D_)))
        if speaker:
            write_hdf5(f, "/speaker_code", np.eye(NS)[i % NS])
        feats.append(f)
    fl, stats = str(tmp_path / "feats.scp"), str(tmp_path / "stats.npz")
    open(fl, "w").write("\n".join(feats) + "\n")
    write_hdf5(stats, "/world/mean", np.zeros(n_aux))
    write_hdf5(stats, "/world/scale", np.ones(n_aux))
    for bs in ("3", "1"):
        outs = {}
        for chunk in ("0", "7"):
            od = str(tmp_path / ("out_bs%s_c%s" % (bs, chunk)))
            _cli(["--feats", fl, "--checkpoint", str(expdir / "checkpoint-final.pkl"), "--stats", stats, "--outdir", od,
                  "--fs", "16000", "--batch_size", bs, "--intervals", "100", "--seed", "5", "--chunk_frames", chunk])
            outs[chunk] = {i: open(os.path.join(od, "c%d.wav" % i), "rb").read() for i in range(3)}
        for i in range(3):
            assert len(outs["0"][i]) > 44 and outs["0"][i] == outs["7"][i], (bs, i)
