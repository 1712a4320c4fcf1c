# -*- coding: utf-8 -*-
"""GPU tier: the warm-up of the bf16 decoder computed in parallel over time (``wnb_decode_bf16_prefill``) is
bit-identical to its sequential warm-up.

Two paths, same inputs, same initial memory (the queues pre-filled with a non-zero byte pattern): (a)
``wnb_decode_bf16_at(pos0 = 0)``, which runs the P - 1 warm-up positions one by one, and (b) the prefill followed by
``wnb_decode_bf16_at(pos0 = P - 1)``.  The generated codes, the teacher-check ``logits_out`` and the whole queue workspace
(padding rows of every cluster included) must be ``torch.equal``, in argmax, supplied-uniform and in-kernel Philox modes
with ragged lengths:
* arctic 512/256 (ks 2, A 28, U 80) at B = 3, 1 (63 padding rows) and 64 (one full cluster); ljspeech-size (ks 3, Ak 128);
  512/512; 256/256 at B = 70 (two clusters of 35); the speaker-code shape (A 31, U 0);
* seeds of one sample, several samples shorter than the receptive field (n_pad > 0), rf + 2 000 and, on a shallow model,
  5 rf + 3 (the prefill computes the pruned windows only and must equal the sequential warm-up over all T0 - 1);
* ``decode_session`` with 1-frame and random chunk schedules equals path (a) and runs the prefill exactly once;
* ``_decode`` at arctic, B = 64, a few hundred Philox samples, equals path (a) and runs the prefill.
That the two paths agree is what says that a wgmma output element depends on its own row of A only: the rows are 64
utterances at one position on path (a) and 64 positions of one utterance on path (b)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

ARCTIC = (256, 28, 512, 256, 10, 3, 2, 80)
LJSPEECH = (256, 80, 512, 256, 10, 1, 3, 256)
R512_S512 = (256, 28, 512, 512, 10, 1, 2, 80)
SHALLOW_256 = (256, 28, 256, 256, 4, 2, 2, 4)
SPEAKER = (256, 31, 256, 256, 4, 2, 2, 0)
_MODELS = {}


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 41 + len(_MODELS))).eval()
        net.decode_math = "bf16"
        _MODELS[t] = (cfg, net)
    return _MODELS[t]


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


def _paths(net, x, h, n_list, mode, uniforms=None, seed=1234, prefill=(False, True)):
    """{prefill: (xs, logits_out, queues)} of one wnb_decode_bf16_at chain per path, from the same inputs and the same
    initial memory"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import MODE_ARGMAX, MODE_SAMPLING, _bf16_prefill, ptr, stream
    lib = _lib.load()
    B, T0 = x.shape
    Q, A, Ap, R, S, ks, U, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                                net.upsampling_factor, len(net.dilations))
    P = max(T0, net.receptive_field)
    n_pad, max_n = P - T0, max(n_list)
    with torch.no_grad():
        w = net._decode_pack()
        wstream = net._decode_bf16_pack()
        upw = net.upsampling.conv.weight.detach().float().contiguous().view(-1) if U > 0 else None
        upb = net.upsampling.conv.bias.detach().float().contiguous().view(-1) if U > 0 else None
    dil = (ctypes.c_int32 * L)(*net.dilations)
    h = h.contiguous().float()
    nsm = torch.tensor(n_list, dtype=torch.int32, device="cuda")
    uni = None if uniforms is None else uniforms.cuda().float().contiguous()
    qbytes = lib.wnb_decode_bf16_workspace(B, R, ks, dil, L)
    cmode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
    out = {}
    for pf in prefill:
        xs = torch.full((B, P + max_n), Q // 2, dtype=torch.int32, device="cuda")
        xs[:, n_pad:P] = x.to(torch.int32)
        queues = torch.full((qbytes,), 0x5A, dtype=torch.uint8, device="cuda")
        lg = torch.full((B, max_n, Q), 7.0, device="cuda")
        if pf:
            _bf16_prefill(lib, xs, P, h, upw, upb, w, wstream, dil, L, queues, n_pad, A, Ap, R, S, ks, U)
        _lib.check(lib.wnb_decode_bf16_at(ptr(xs), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]), ptr(wstream),
                                          dil, L, ptr(queues), ptr(nsm), ptr(uni), ptr(lg), B, P, max_n, n_pad,
                                          h.size(2), Q, A, Ap, R, S, ks, U, cmode, ctypes.c_uint64(seed),
                                          P - 1 if pf else 0, 0, 0, stream()),
                   "decode_bf16_at")
        torch.cuda.synchronize()
        out[pf] = (xs.cpu(), lg.cpu(), queues.cpu())
    return out


def _count_prefills(monkeypatch):
    """wrap nets.wavenet._bf16_prefill so that a test can check the Python layer does run it"""
    from pytorchwavenetvocoder_b200.nets import wavenet
    calls = []
    real = wavenet._bf16_prefill

    def counted(*args):
        calls.append(args[2])   # P
        return real(*args)
    monkeypatch.setattr(wavenet, "_bf16_prefill", counted)
    return calls


def _assert_equal(out, what):
    (xa, la, qa), (xb, lb, qb) = out[False], out[True]
    assert torch.equal(qa, qb), ("queues", what, int((qa != qb).sum()), qa.numel())
    assert torch.equal(la, lb), ("logits", what)
    assert torch.equal(xa, xb), ("codes", what)


# id: (model, B, T0 as a function of the receptive field)
CASES = {
    "shallow_256_B70": (SHALLOW_256, 70, lambda rf: 1),
    "arctic_B3": (ARCTIC, 3, lambda rf: 1),
    "ljspeech_ks3": (LJSPEECH, 3, lambda rf: 1),
    "r512_s512": (R512_S512, 4, lambda rf: 1),
    "arctic_B1": (ARCTIC, 1, lambda rf: 1),
    "arctic_B64": (ARCTIC, 64, lambda rf: 1),
    "speaker_A31_U0": (SPEAKER, 5, lambda rf: 1),
    "arctic_multi_sample_seed": (ARCTIC, 3, lambda rf: 517),      # n_pad = rf - 517
    "shallow_multi_sample_seed": (SHALLOW_256, 5, lambda rf: 9),
    "arctic_rf_plus_2000": (ARCTIC, 3, lambda rf: rf + 2000),
    "shallow_5rf": (SHALLOW_256, 5, lambda rf: 5 * rf + 3),
}


@pytest.mark.parametrize("case", list(CASES))
def test_prefill_equals_sequential_warmup(case):
    t, B, t0fn = CASES[case]
    cfg, net = _model(t)
    T0 = t0fn(cfg.receptive_field)
    max_n = 40
    ci = list(CASES).index(case)
    x, h, n_list = _inputs(cfg, B, T0, max_n, 100 + ci)
    uni = torch.from_numpy(np.random.RandomState(ci).uniform(size=(B, max_n)).astype(np.float32))
    _assert_equal(_paths(net, x, h, n_list, "argmax"), (case, "argmax"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", uniforms=uni), (case, "uniforms"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=1000 + ci), (case, "philox"))


@pytest.mark.parametrize("sched", ["ones", "random"])
@pytest.mark.parametrize("t", [SHALLOW_256, ARCTIC], ids=["shallow", "arctic"])
def test_session_equals_sequential_path(sched, t, monkeypatch):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    cfg, net = _model(t)
    B, max_n = 3, 200
    x, h, n_list = _inputs(cfg, B, 1, max_n, 11)
    want_xs, want_lg, _ = _paths(net, x, h, n_list, "sampling", seed=5, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    rng = np.random.RandomState(3)
    with torch.no_grad():
        s = DecodeSession(net, x, n_list, "sampling", 5, None, True, "bf16")
        codes, logits = [[] for _ in range(B)], [[] for _ in range(B)]
        f0 = 0
        while not s.done:
            F = 1 if sched == "ones" else int(rng.randint(1, 6))
            gen, lg = s.step(h[:, :, f0:f0 + F])
            f0 += F
            for b, c in enumerate(s.last_counts):
                codes[b].append(gen[b, :c].cpu())
                logits[b].append(lg[b, :c].cpu())
    assert s.kernel == "bf16"
    P = cfg.receptive_field
    assert prefills == [P]   # the call that reached sample 0 ran the warm-up as a prefill, and no other call did
    for b, n in enumerate(n_list):
        assert torch.equal(torch.cat(codes[b]), want_xs[b, P:P + n]), b
        assert torch.equal(torch.cat(logits[b]), want_lg[b, :n]), b


def test_arctic_decode_equals_sequential(monkeypatch):
    cfg, net = _model(ARCTIC)
    B, n = 64, 300
    x, h, _ = _inputs(cfg, B, 1, n, 21)
    n_list = [n] * B
    want_xs, _, _ = _paths(net, x, h, n_list, "sampling", seed=1234, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    with torch.no_grad():
        gen = net._decode(x, h, n_list, "sampling", seed=1234)
    assert net.last_decode_kernel == "bf16"
    P = cfg.receptive_field
    assert prefills == [P]
    assert torch.equal(gen.cpu(), want_xs[:, P:])
