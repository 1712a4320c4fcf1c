# -*- coding: utf-8 -*-
"""GPU tier: the decode warm-up computed in parallel over time (``wnb_decode_warp_prefill``) is bit-identical to the
sequential warm-up.

Two paths, same inputs, same initial queue memory: (a) ``wnb_decode_warp_at(pos0 = 0)``, which runs the P - 1 warm-up
positions one by one, and (b) the prefill followed by ``wnb_decode_warp_at(pos0 = P - 1)``.  The generated codes, the
teacher-check ``logits_out`` and the whole queue workspace must be ``torch.equal``:
* all eight ``decode_warp_kernel`` forms (reached as in test_gpu_decode_forms.py and asserted through
  ``wnb_decode_warp_form``) and the speaker-code shape (U = 0, A = 31); argmax, supplied uniforms and in-kernel Philox;
  ragged lengths; one- and multi-sample seeds;
* seeds longer than the receptive field (rf + 2 000 at the bench shape, 5 rf + 3 at a shallow one): the prefill computes
  the last rf - 1 positions only and must equal the sequential warm-up over all T0 - 1;
* ``decode_session`` with 1-frame and random chunk schedules equals path (a), and runs the prefill exactly once;
* ``_decode`` at the bench shape, B = 64, 2 000 Philox samples, equals path (a), and runs the prefill."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

SHALLOW = (256, 28, 64, 512, 4, 2, 2, 4)      # L = 8, largest dilation 8
BENCH = (256, 28, 64, 512, 10, 3, 2, 80)      # the bench's decode shape
_MODELS = {}


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        _MODELS[t] = (cfg, our_model(cfg, O.make_params(cfg, 41 + len(_MODELS))).eval())
    return _MODELS[t]


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


def _paths(net, x, h, n_list, mode, uniforms=None, seed=1234, prefill=(False, True)):
    """{prefill: (xs, logits_out, queues)} of one wnb_decode_warp_at chain per path, from the same inputs and the same
    initial memory (a finite fill, so that untouched slots compare equal)"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import MODE_ARGMAX, MODE_SAMPLING, _warp_prefill, ptr, stream
    lib = _lib.load()
    B, T0 = x.shape
    Q, A, U, L = net.n_quantize, net.n_aux, net.upsampling_factor, len(net.dilations)
    P = max(T0, net.receptive_field)
    n_pad, max_n = P - T0, max(n_list)
    with torch.no_grad():
        w = net._decode_pack()
        W, CL = lib.wnb_decode_warp_plan(B), lib.wnb_decode_warp_cluster(B)
        wstream = net._decode_warp_pack(W, CL)
        upw = net.upsampling.conv.weight.detach().float().contiguous().view(-1) if U > 0 else None
        upb = net.upsampling.conv.bias.detach().float().contiguous().view(-1) if U > 0 else None
    dil = (ctypes.c_int32 * L)(*net.dilations)
    h = h.contiguous().float()
    nsm = torch.tensor(n_list, dtype=torch.int32, device="cuda")
    uni = None if uniforms is None else uniforms.cuda().float().contiguous()
    qn = lib.wnb_decode_workspace(B, 64, 2, dil, L) // 4
    cmode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
    out = {}
    for pf in prefill:
        xs = torch.full((B, P + max_n), Q // 2, dtype=torch.int32, device="cuda")
        xs[:, n_pad:P] = x.to(torch.int32)
        queues = torch.full((qn,), 7.0, device="cuda")
        lg = torch.full((B, max_n, Q), 7.0, device="cuda")
        if pf:
            _warp_prefill(lib, xs, P, h, upw, upb, w, dil, L, queues, n_pad, A, U, CL)
        _lib.check(lib.wnb_decode_warp_at(ptr(xs), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]), ptr(wstream),
                                          ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), dil, L, ptr(queues),
                                          ptr(nsm), ptr(uni), ptr(lg), B, P, max_n, n_pad, h.size(2), A, U, cmode,
                                          ctypes.c_uint64(seed), W, CL, P - 1 if pf else 0, 0, 0, stream()),
                   "decode_warp_at")
        torch.cuda.synchronize()
        out[pf] = (xs.cpu(), lg.cpu(), queues.cpu())
    return out


def _count_prefills(monkeypatch):
    """wrap nets.wavenet._warp_prefill so that a test can check the Python layer does run it"""
    from pytorchwavenetvocoder_b200.nets import wavenet
    calls = []
    real = wavenet._warp_prefill

    def counted(*args):
        calls.append(args[2])   # P
        return real(*args)
    monkeypatch.setattr(wavenet, "_warp_prefill", counted)
    return calls


def _assert_equal(out, what):
    (xa, la, qa), (xb, lb, qb) = out[False], out[True]
    assert torch.equal(xa, xb), ("codes", what)
    assert torch.equal(la, lb), ("logits", what)
    assert torch.equal(qa, qb), ("queues", what, int((qa != qb).sum()))


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
def test_prefill_equals_sequential_warmup_every_form(form_id, monkeypatch):
    t, bfn, big, want = WARP_FORMS[form_id]
    if big is not None:
        monkeypatch.setenv("WNB_DECODE_BIG", big)
    cfg, net = _model(t)
    B = bfn(_nsm())
    assert _warp_form(B, len(cfg.dilations)) == want
    ci = list(WARP_FORMS).index(form_id)
    T0 = 1 if ci % 2 == 0 else 1 + ci * 3          # one-sample and multi-sample seeds
    max_n = 48
    x, h, n_list = _inputs(cfg, B, T0, max_n, 100 + ci)
    uni = torch.from_numpy(np.random.RandomState(ci).uniform(size=(B, max_n)).astype(np.float32))
    _assert_equal(_paths(net, x, h, n_list, "argmax"), (form_id, "argmax"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", uniforms=uni), (form_id, "uniforms"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=1000 + ci), (form_id, "philox"))


@pytest.mark.parametrize("case", ["bench_rf_plus_2000", "shallow_5rf"])
def test_prefill_long_seed(case):
    t, B = (BENCH, 3) if case == "bench_rf_plus_2000" else (SHALLOW, 5)
    cfg, net = _model(t)
    rf = cfg.receptive_field
    T0 = rf + 2000 if case == "bench_rf_plus_2000" else 5 * rf + 3
    x, h, n_list = _inputs(cfg, B, T0, 40, 7)
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=99), (case, "philox"))
    _assert_equal(_paths(net, x, h, n_list, "argmax"), (case, "argmax"))


@pytest.mark.parametrize("sched", ["ones", "random"])
@pytest.mark.parametrize("t", [SHALLOW, BENCH], ids=["shallow", "bench"])
def test_session_equals_sequential_path(sched, t, monkeypatch):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    cfg, net = _model(t)
    B, max_n = 3, 120
    x, h, n_list = _inputs(cfg, B, 1, max_n, 11)
    want_xs, want_lg, _ = _paths(net, x, h, n_list, "sampling", seed=5, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    rng = np.random.RandomState(3)
    with torch.no_grad():
        s = DecodeSession(net, x, n_list, "sampling", 5, None, True, "warp")
        codes, logits = [[] for _ in range(B)], [[] for _ in range(B)]
        f0 = 0
        while not s.done:
            F = 1 if sched == "ones" else int(rng.randint(1, 6))
            gen, lg = s.step(h[:, :, f0:f0 + F])
            f0 += F
            for b, c in enumerate(s.last_counts):
                codes[b].append(gen[b, :c].cpu())
                logits[b].append(lg[b, :c].cpu())
    assert s.kernel == "warp"
    P = max(1, cfg.receptive_field)
    assert prefills == [P]   # the call that reached sample 0 ran the warm-up as a prefill, and no other call did
    for b, n in enumerate(n_list):
        assert torch.equal(torch.cat(codes[b]), want_xs[b, P:P + n]), b
        assert torch.equal(torch.cat(logits[b]), want_lg[b, :n]), b


def test_bench_shape_decode_equals_sequential(monkeypatch):
    cfg, net = _model(BENCH)
    B, n = 64, 2000
    x, h, _ = _inputs(cfg, B, 1, n, 21)
    n_list = [n] * B
    want_xs, _, _ = _paths(net, x, h, n_list, "sampling", seed=1234, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    with torch.no_grad():
        gen = net._decode(x, h, n_list, "sampling", seed=1234)
    assert net.last_decode_kernel == "warp"
    P = cfg.receptive_field
    assert prefills == [P]
    assert torch.equal(gen.cpu(), want_xs[:, P:])
