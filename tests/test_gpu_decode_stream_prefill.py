# -*- coding: utf-8 -*-
"""GPU tier: the streaming decoder's warm-up computed in parallel over time (``wnb_decode_stream_prefill``) is
bit-identical to its sequential warm-up.

Two paths, same inputs, same initial queue memory: (a) ``wnb_decode_stream_at(pos0 = 0)``, which runs the P - 1 warm-up
positions one by one, and (b) the prefill followed by ``wnb_decode_stream_at(pos0 = P - 1)``.  The generated codes, the
teacher-check ``logits_out`` and the whole queue workspace must be ``torch.equal``:
* 64/64 at ks 2 and ks 3, with and without an up-sampling layer; the speaker-code shape (U 0, A 31); n_quantize 64;
  dilations that are not powers of two; arctic 512/256 ks 2 U 80 and ljspeech-melspc 512/256 ks 3 U 256 (few samples);
* B = 1, B > SMs and B > 2 SMs (the decoder's NU 1, 2 and 4; the prefill's groups of 64 rows);
* argmax, supplied uniforms and in-kernel Philox; one-sample seeds, seeds longer than the pruned window, ragged lengths;
* ``decode_session`` on the streaming kernel, fed in chunks, equals path (a) and runs the prefill exactly once;
* a one-shot decode on the streaming kernel makes L + 1 launches (the prefill's front and L - 1 layers, and the decode)
  at a shape outside the warp decoder, and one sequential launch when "stream" is named at a shape the warp decoder
  covers."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

KS2_U = (256, 28, 64, 64, 4, 2, 2, 4)
KS3_U = (256, 28, 64, 64, 4, 2, 3, 4)
KS3_U0 = (256, 28, 64, 64, 4, 2, 3, 0)
SPEAKER = (256, 31, 64, 64, 4, 2, 2, 0)
Q64 = (64, 28, 64, 64, 3, 2, 2, 4)
ARCTIC = (256, 28, 512, 256, 10, 3, 2, 80)
LJ_MELSPC = (256, 80, 512, 256, 10, 3, 3, 256)
ODD_DIL = [3, 1, 5, 2, 7, 6, 1, 4]      # replaces KS3_U's 8 power-of-two dilations
_MODELS = {}


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _model(t, dil=None):
    key = (t, tuple(dil or ()))
    if key not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 61 + len(_MODELS))).eval()
        if dil is not None:   # the weights do not depend on the dilations; the decoders take them as a list
            assert len(dil) == len(net.dilations)
            net.dilations = list(dil)
            net.receptive_field = (net.kernel_size - 1) * sum(dil) + 1
        _MODELS[key] = net
    return _MODELS[key]


def _inputs(net, B, T0, max_n, seed):
    rng = np.random.RandomState(seed)
    U = max(net.upsampling_factor, 1)
    P = max(T0, net.receptive_field)
    x = torch.from_numpy(rng.randint(0, net.n_quantize, size=(B, T0))).cuda()
    h = torch.from_numpy(rng.standard_normal((B, net.n_aux, (P + max_n + U - 1) // U + 1)).astype(np.float32)).cuda()
    n_list = [int(v) for v in rng.randint(1, max_n + 1, size=B)]
    n_list[0] = 1
    if B > 1:
        n_list[1] = max_n
    return x, h, n_list


def _paths(net, x, h, n_list, mode, uniforms=None, seed=1234, prefill=(False, True)):
    """{prefill: (xs, logits_out, queues)} of one wnb_decode_stream_at chain per path, from the same inputs and the same
    initial memory (a finite fill, so that untouched slots compare equal)"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import (MODE_ARGMAX, MODE_SAMPLING, _decode_snapshot, _stream_prefill,
                                                         ptr, stream)
    lib = _lib.load()
    B, T0 = x.shape
    Q, A, Ap, R, S, ks, U, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                                net.upsampling_factor, len(net.dilations))
    assert lib.wnb_decode_stream_supported(Q, Ap, R, S, ks, L)
    P = max(T0, net.receptive_field)
    n_pad, max_n = P - T0, max(n_list)
    with torch.no_grad():
        w, upw, upb = _decode_snapshot(net)
        wstream = net._decode_stream_pack(w)
    dil = (ctypes.c_int32 * L)(*net.dilations)
    h = h.contiguous().float()
    nsm = torch.tensor(n_list, dtype=torch.int32, device="cuda")
    uni = None if uniforms is None else uniforms.cuda().float().contiguous()
    qn = lib.wnb_decode_workspace(B, R, ks, dil, L) // 4
    cmode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
    out = {}
    for pf in prefill:
        xs = torch.full((B, P + max_n), Q // 2, dtype=torch.int32, device="cuda")
        xs[:, n_pad:P] = x.to(torch.int32)
        queues = torch.full((qn,), 7.0, device="cuda")
        lg = torch.full((B, max_n, Q), 7.0, device="cuda")
        if pf:
            _stream_prefill(lib, xs, P, h, upw, upb, w, wstream, dil, L, queues, n_pad, Q, A, Ap, R, S, ks, U)
        _lib.check(lib.wnb_decode_stream_at(ptr(xs), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]),
                                            ptr(wstream), ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), dil,
                                            L, ptr(queues), ptr(nsm), ptr(uni), ptr(lg), B, P, max_n, n_pad, h.size(2),
                                            Q, A, Ap, R, S, ks, U, cmode, ctypes.c_uint64(seed), P - 1 if pf else 0, 0,
                                            0, stream()),
                   "decode_stream_at")
        torch.cuda.synchronize()
        out[pf] = (xs.cpu(), lg.cpu(), queues.cpu())
    return out


def _count_prefills(monkeypatch):
    """wrap nets.wavenet._stream_prefill so that a test can check the Python layer does run it"""
    from pytorchwavenetvocoder_b200.nets import wavenet
    calls = []
    real = wavenet._stream_prefill

    def counted(*args):
        calls.append(args[2])   # P
        return real(*args)
    monkeypatch.setattr(wavenet, "_stream_prefill", counted)
    return calls


def _assert_equal(out, what):
    (xa, la, qa), (xb, lb, qb) = out[False], out[True]
    assert torch.equal(xa, xb), ("codes", what)
    assert torch.equal(la, lb), ("logits", what)
    assert torch.equal(qa, qb), ("queues", what, int((qa != qb).sum()))


SMALL = {"ks2_u4": KS2_U, "ks3_u4": KS3_U, "ks3_u0": KS3_U0, "speaker_A31_U0": SPEAKER, "q64": Q64,
         "odd_dilations": KS3_U}


@pytest.mark.parametrize("shape", list(SMALL))
def test_prefill_equals_sequential_warmup(shape):
    net = _model(SMALL[shape], ODD_DIL if shape == "odd_dilations" else None)
    si = list(SMALL).index(shape)
    B, max_n = 5, 40
    for T0 in (1, 3 * net.receptive_field + 5):     # a one-sample seed, and one longer than the pruned window
        x, h, n_list = _inputs(net, B, T0, max_n, 100 + si)
        uni = torch.from_numpy(np.random.RandomState(si).uniform(size=(B, max_n)).astype(np.float32))
        _assert_equal(_paths(net, x, h, n_list, "argmax"), (shape, T0, "argmax"))
        _assert_equal(_paths(net, x, h, n_list, "sampling", uniforms=uni), (shape, T0, "uniforms"))
        _assert_equal(_paths(net, x, h, n_list, "sampling", seed=1000 + si), (shape, T0, "philox"))


@pytest.mark.parametrize("rows", ["one", "sms_plus", "two_sms_plus"])
def test_prefill_every_decoder_form(rows):
    """B = 1, sms + 3 and 2 sms + 5 rows: the decoder runs NU 1, 2 and 4; the prefill groups rows by 64"""
    net = _model(KS2_U)
    B = {"one": 1, "sms_plus": _nsm() + 3, "two_sms_plus": 2 * _nsm() + 5}[rows]
    x, h, n_list = _inputs(net, B, 7, 24, 7)
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=99), (rows, "philox"))
    _assert_equal(_paths(net, x, h, n_list, "argmax"), (rows, "argmax"))


@pytest.mark.parametrize("shape", ["arctic", "ljspeech_melspc"])
def test_prefill_recipe_shapes(shape):
    net = _model(ARCTIC if shape == "arctic" else LJ_MELSPC)
    x, h, n_list = _inputs(net, 2, 1, 6, 3)
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=5), (shape, "philox"))


@pytest.mark.parametrize("sched", ["ones", "random"])
def test_session_equals_sequential_path(sched, monkeypatch):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    net = _model(KS3_U)
    B, max_n = 3, 120
    x, h, n_list = _inputs(net, B, 1, max_n, 11)
    want_xs, want_lg, _ = _paths(net, x, h, n_list, "sampling", seed=5, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    rng = np.random.RandomState(3)
    with torch.no_grad():
        s = DecodeSession(net, x, n_list, "sampling", 5, None, True, "stream")
        codes, logits = [[] for _ in range(B)], [[] for _ in range(B)]
        f0 = 0
        while not s.done:
            F = 1 if sched == "ones" else int(rng.randint(1, 6))
            gen, lg = s.step(h[:, :, f0:f0 + F])
            f0 += F
            for b, c in enumerate(s.last_counts):
                codes[b].append(gen[b, :c].cpu())
                logits[b].append(lg[b, :c].cpu())
    assert s.kernel == "stream"
    P = net.receptive_field
    assert prefills == [P]   # the call that reached sample 0 ran the warm-up as a prefill, and no other call did
    for b, n in enumerate(n_list):
        assert torch.equal(torch.cat(codes[b]), want_xs[b, P:P + n]), b
        assert torch.equal(torch.cat(logits[b]), want_lg[b, :n]), b


def test_auto_one_shot_picks_stream_and_prefills(monkeypatch):
    """fp32 "auto" on a shape outside the warp decoder runs the streaming decoder with its prefill, and decodes what the
    sequential path decodes"""
    net = _model(KS3_U)
    x, h, n_list = _inputs(net, 4, 1, 50, 21)
    want_xs, _, _ = _paths(net, x, h, n_list, "sampling", seed=77, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    with torch.no_grad():
        gen = net._decode(x, h, n_list, "sampling", seed=77)
    assert net.last_decode_kernel == "stream" and prefills == [net.receptive_field]
    P = net.receptive_field
    for b, n in enumerate(n_list):
        assert torch.equal(gen[b, :n].cpu(), want_xs[b, P:P + n]), b


WARP_SHAPE = (256, 28, 64, 512, 4, 2, 2, 4)    # covered by the warp decoder: "stream" runs there only when named


@pytest.mark.parametrize("case", ["stream_ks2", "stream_ks3_auto", "stream_named_at_warp_shape"])
def test_oneshot_launch_count(case, monkeypatch):
    """L + 1 launches (the prefill's front and L - 1 layers, then the decode) on a shape outside the warp decoder; one
    sequential decode launch when "stream" is named at a shape the warp decoder covers"""
    from pytorchwavenetvocoder_b200 import _lib
    net, kernel = {"stream_ks2": (_model(KS2_U), "stream"), "stream_ks3_auto": (_model(KS3_U), "auto"),
                   "stream_named_at_warp_shape": (_model(WARP_SHAPE), "stream")}[case]
    x, h, n_list = _inputs(net, 5, 1, 8, 900)
    want_xs, _, _ = _paths(net, x, h, n_list, "sampling", seed=3, prefill=(False,))[False]
    prefills = _count_prefills(monkeypatch)
    l0 = _lib.launch_count()
    with torch.no_grad():
        gen = net._decode(x, h, n_list, "sampling", seed=3, kernel=kernel)
    launches = _lib.launch_count() - l0
    assert net.last_decode_kernel == "stream"
    parallel = case != "stream_named_at_warp_shape"
    assert launches == (len(net.dilations) + 1 if parallel else 1), (case, launches)
    assert prefills == ([net.receptive_field] if parallel else []), case
    P = net.receptive_field
    for b, n in enumerate(n_list):
        assert torch.equal(gen[b, :n].cpu(), want_xs[b, P:P + n]), (case, b)
