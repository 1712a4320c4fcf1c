# -*- coding: utf-8 -*-
"""GPU tier: continuous batching on the bf16 decoder (``WaveNet.decode_pool``) is bit-identical to one-shot decoding.

Every case admits about 80 streams at staggered calls into a pool of capacity 8 (many admissions into reused rows), 64
(one cluster) or 130 (three clusters), with seeds of one sample, rf + 2 000 and 5 rf + 3 mixed in one pool, lengths of
50-400 samples, aux frames in random chunks and random ``max_samples`` windows that split streams across calls.  Stream
k of a pool with seed S must equal row k of ``net._decode(X, H, n_list, mode, seed=S, kernel="bf16")`` (``torch.equal``)
in argmax and in Philox sampling, on arctic 512/256, the ljspeech-size shape (ks 3, Ak 128), 256/256 with 8 layers and
the speaker-code shape (U 0, A 31); one run lowers ``POOL_COUNTER_LIMIT`` so that the counter rebases mid-stream.  Also:
the uniforms kernel against ``tests/decode_reference.py::philox_uniform`` bit for bit, ``step_pcm16``, the errors, and
the library launches of a steady, an admitting and an empty call."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.decode_reference import philox_uniform
from tests.util import our_model

pytestmark = pytest.mark.gpu

ARCTIC = (256, 28, 512, 256, 10, 3, 2, 80)
LJSPEECH = (256, 80, 512, 256, 10, 1, 3, 256)
SHALLOW_256 = (256, 28, 256, 256, 4, 2, 2, 4)
SPEAKER = (256, 31, 256, 256, 4, 2, 2, 0)
_MODELS = {}


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 61 + len(_MODELS))).eval()
        net.decode_math = "bf16"
        _MODELS[t] = (cfg, net)
    return _MODELS[t]


def _streams(cfg, n, seed):
    """n streams: seed codes, length, aux frames (A, nf) on the GPU, arrival call"""
    rng = np.random.RandomState(seed)
    rf, U = cfg.receptive_field, max(cfg.upsampling_factor, 1)
    out = []
    for k in range(n):
        T0 = [1, rf + 2000, 5 * rf + 3][k % 3]
        total = int(rng.randint(50, 401))
        nf = (T0 - 1 + total + U - 1) // U + 1
        x = torch.from_numpy(rng.randint(0, cfg.n_quantize, size=T0)).cuda()
        h = torch.from_numpy(rng.standard_normal((cfg.n_aux, nf)).astype(np.float32)).cuda()
        out.append((x, total, h, int(rng.randint(0, 40))))
    return out


def _one_shot(net, streams, mode, seed):
    """{k: codes of stream k} from one-shot bf16 decodes, one per seed length, stream k in row k"""
    want = {}
    N, A, U = len(streams), net.n_aux, max(net.upsampling_factor, 1)
    # one batch: frames for the longest seed and the longest length (a row reads its own frames only)
    nfmax = (max(x.numel() for x, _, _, _ in streams) - 1 + max(n for _, n, _, _ in streams) + U - 1) // U + 1
    H = torch.zeros(N, A, nfmax, device="cuda")
    for k, (_, _, h, _) in enumerate(streams):
        H[k, :, :h.size(1)] = h
    n_list = [total for _, total, _, _ in streams]
    for T0 in sorted({x.numel() for x, _, _, _ in streams}):
        X = torch.zeros(N, T0, dtype=torch.int64, device="cuda")
        for k, (x, _, _, _) in enumerate(streams):
            if x.numel() == T0:
                X[k] = x
        with torch.no_grad():
            gen = net._decode(X, H, n_list, mode, seed=seed, kernel="bf16").cpu()
        for k, (x, total, _, _) in enumerate(streams):
            if x.numel() == T0:
                want[k] = gen[k, :total]
    return want


def _run_pool(net, streams, capacity, mode, seed, rng_seed):
    rng = np.random.RandomState(rng_seed)
    pool = net.decode_pool(capacity, mode, seed)
    got = {k: [] for k in range(len(streams))}
    sent = [0] * len(streams)
    it = 0
    while it <= max(a for _, _, _, a in streams) or not all(pool.finished(k) for k in range(len(streams))):
        for k, (x, total, h, arrival) in enumerate(streams):
            if arrival == it:
                F = int(rng.randint(0, 3))
                assert pool.admit(x, total, h[:, :F] if F else None, stream=k) == k
                sent[k] = F
            elif arrival < it and not pool.finished(k) and sent[k] < h.size(1):
                F = min(int(rng.randint(0, 40)), h.size(1) - sent[k])
                pool.feed(k, h[:, sent[k]:sent[k] + F])
                sent[k] += F
        it += 1
        for k, codes in pool.step(None if rng.rand() < 0.2 else int(rng.randint(1, 150))).items():
            got[k].append(codes.cpu())
    return pool, {k: torch.cat(v) for k, v in got.items()}


CASES = {
    "arctic": ARCTIC,
    "ljspeech_ks3": LJSPEECH,
    "r256_L8": SHALLOW_256,
    "speaker_A31_U0": SPEAKER,
}


@pytest.mark.parametrize("capacity", [8, 64, 130])
@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("case", list(CASES))
def test_pool_equals_one_shot(case, mode, capacity):
    cfg, net = _model(CASES[case])
    ci = list(CASES).index(case)
    streams = _streams(cfg, 80, 10 * ci + capacity)
    seed = 1000 + ci
    want = _one_shot(net, streams, mode, seed)
    pool, got = _run_pool(net, streams, capacity, mode, seed, 7 * ci + capacity)
    assert not pool.active and not pool.waiting
    for k in range(len(streams)):
        assert torch.equal(got[k], want[k]), (case, mode, capacity, k, int((got[k] != want[k]).sum()))


def test_counter_rebase_mid_stream(monkeypatch):
    from pytorchwavenetvocoder_b200.nets import wavenet
    cfg, net = _model(SHALLOW_256)
    streams = _streams(cfg, 40, 77)
    want = _one_shot(net, streams, "sampling", 9)
    period = 8   # lcm of the queue lengths 1, 2, 4, 8
    monkeypatch.setattr(wavenet, "POOL_COUNTER_LIMIT", 1 + period + 257)
    g0s = []
    real = wavenet.PoolSchedule.next_call

    def traced(self, max_samples=None):
        call = real(self, max_samples)
        if call is not None:
            g0s.append(call.g0)
        return call
    monkeypatch.setattr(wavenet.PoolSchedule, "next_call", traced)
    _, got = _run_pool(net, streams, 8, "sampling", 9, 5)
    assert sum(b < a for a, b in zip(g0s, g0s[1:])) >= 3, g0s
    for k in range(len(streams)):
        assert torch.equal(got[k], want[k]), k


def test_uniforms_kernel_equals_philox_uniform():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import ptr, stream
    lib = _lib.load()
    B, A, F, n, U = 5, 3, 4, 300, 80
    seed = 0x0123456789ABCDEF
    sample0, sid, count = [0, 7, 2 ** 20, 5, 123456789], [0, 1, 99, 2 ** 31 - 1, 12], [n, 17, n, 0, 1]
    table = torch.tensor([[0] * B, [0] * B, sample0, sid, count], dtype=torch.int32, device="cuda")
    frames = torch.randn(B, A, F, device="cuda")
    upw, upb = torch.randn(U, device="cuda"), torch.randn(1, device="cuda")
    aux = torch.full((B, A, n), 7.0, device="cuda")
    uni = torch.full((B, n), 7.0, device="cuda")
    _lib.check(lib.wnb_decode_bf16_pool_inputs(ptr(frames), ptr(upw), ptr(upb), ptr(table), ptr(aux), ptr(uni), B, A, F,
                                               n, U, ctypes.c_uint64(seed), stream()), "pool_inputs")
    got = uni.cpu().numpy()
    for b in range(B):
        want = philox_uniform(seed, sid[b], np.arange(sample0[b], sample0[b] + count[b]))
        assert np.array_equal(got[b, :count[b]], want), b
        assert (got[b, count[b]:] == 0).all(), b


def test_step_pcm16_equals_codes():
    from pytorchwavenetvocoder_b200.nets.wavenet import codes_to_pcm16
    cfg, net = _model(SHALLOW_256)
    streams = _streams(cfg, 3, 5)
    want = _one_shot(net, streams, "sampling", 4)
    pool = net.decode_pool(4, "sampling", 4)
    got = {k: [] for k in range(3)}
    for k, (x, total, h, _) in enumerate(streams):
        pool.admit(x, total, h)
    while pool.active or pool.waiting:
        for k, pcm in pool.step_pcm16(64).items():
            got[k].append(pcm.cpu())
    for k in range(3):
        assert torch.equal(torch.cat(got[k]), codes_to_pcm16(want[k].cuda(), 256).cpu()), k


def test_errors():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import WaveNet
    cfg, net = _model(SHALLOW_256)
    net.decode_math = "fp32"
    try:
        with pytest.raises(_lib.WnbError):
            net.decode_pool(8)
    finally:
        net.decode_math = "bf16"
    small = WaveNet(256, 28, 64, 512, 3, 1, 2, 4).cuda()             # 64/512: outside the bf16 decoder
    small.decode_math = "bf16"
    with pytest.raises(_lib.WnbError):
        small.decode_pool(8)
    pool = net.decode_pool(8, "argmax")
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    with pytest.raises(_lib.WnbError):
        pool.admit(x.cpu(), 10)
    sid = pool.admit(x, 10)
    with pytest.raises(_lib.WnbError):
        pool.feed(sid, torch.zeros(28, 3))
    with pytest.raises(ValueError):
        pool.feed(sid, torch.zeros(27, 3, device="cuda"))
    with pytest.raises(ValueError):
        pool.feed(sid, torch.zeros(1, 28, 3, device="cuda"))
    with pytest.raises(KeyError):
        pool.feed(sid + 1, torch.zeros(28, 3, device="cuda"))
    with pytest.raises(KeyError):
        pool.finished(sid + 1)
    with pytest.raises(ValueError):
        pool.admit(x, 10, stream=sid)                                 # the id exists already
    with pytest.raises(ValueError):
        pool.admit(x, 0)
    with pytest.raises(ValueError):
        net.decode_pool(0)


def test_launch_counts():
    """steady call: the inputs kernel and the decode; admitting call (one seed length, 8 layers): the prefill's front and
    7 x (gate, res), the transplant, the inputs kernel and the decode; a call with no runnable stream: nothing"""
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = _model(SHALLOW_256)
    pool = net.decode_pool(8, "sampling", 3)
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    h = torch.randn(28, 40, device="cuda")
    pool.admit(x, 100, h[:, :10])
    pool.admit(x, 100, h[:, :10])
    counts = []
    for _ in range(3):
        l0 = _lib.launch_count()
        out = pool.step()
        counts.append((_lib.launch_count() - l0, sorted(out)))
    torch.cuda.synchronize()
    # the first call admits both streams in one prefill; 10 frames of U 4 are samples 0 .. 39, so the second call has
    # nothing to run
    assert counts == [(18, [0, 1]), (0, []), (0, [])], counts
    pool.feed(0, h[:, 10:20])
    pool.feed(1, h[:, 10:20])
    l0 = _lib.launch_count()
    out = pool.step()
    assert _lib.launch_count() - l0 == 2 and sorted(out) == [0, 1] and out[0].numel() == 40
