# -*- coding: utf-8 -*-
"""GPU tier: the bf16 decoder (csrc/decode_bf16.cu) layer by layer against float64, teacher-forced from its own
dilation queues (tests/decode_bf16_layers.py).

Driver.  The warm-up runs as ``DecodeSession.step`` runs it (``_bf16_prefill``), then one ``wnb_decode_bf16_at`` call
per position: max_n = 1, pos0 = P - 1 + i, the window arguments ``DecodeSession.step`` builds, n_samples 1 or 0 per row
(ragged lengths, 1 among them; every cluster keeps one full-length row, because a cluster whose rows have all finished
stops and leaves its queues as they are).  Before the first call the whole queue workspace is read once, which gives every
layer's last (ks-1) d_l positions; after each call the newest slot of every layer.  Every padding row of a cluster must
equal the cluster's last utterance in every slot read.

Guard.  The chained codes and ``logits_out`` must ``torch.equal`` a one-shot ``net._decode`` with the same seed and
mode: this shows the driver runs the decoder's normal path, and it carries the check over to multi-step launches (a
one-position call sends every d = 1 tap across a launch boundary; only the one-shot launch uses the in-kernel step
barrier).

Every case runs in argmax mode and with in-kernel Philox sampling, over a window of 24 positions in which every layer's
slot index wraps (a one-sample seed puts P - 1 just below a multiple of every queue length), plus one case after a
seed of rf + 2 000 samples.  The largest ratio of every observable is printed (and written as decode_bf16_layers_*.json
when $WNB_PARITY_OUT is set)."""
import ctypes
import json
import os
import time

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests import decode_bf16_layers as DL
from tests.util import our_model

pytestmark = pytest.mark.gpu

N = 24
# id: ((Q, A, R, S, depth, repeat, ks, U), B, T0 as a function of the receptive field)
CASES = {
    "arctic": ((256, 28, 512, 256, 10, 3, 2, 80), 3, lambda rf: 1),          # L 30, d <= 512, 61 padding rows
    "ks3": ((256, 80, 512, 256, 10, 1, 3, 256), 3, lambda rf: 1),            # two taps, queues of 2d, Ak 128
    "r512_s512": ((256, 28, 512, 512, 10, 1, 2, 80), 4, lambda rf: 1),       # decode_bf16_kernel<512, 512>
    "wide_aux": ((256, 256, 256, 256, 4, 2, 3, 0), 65, lambda rf: 1),        # Ak 256, ks 3 at R 256, clusters 33 + 32
    "deep": ((256, 28, 256, 256, 4, 16, 2, 4), 64, lambda rf: 1),            # L 64 = kMaxL, one full cluster
    "speaker": ((256, 31, 256, 256, 4, 2, 2, 0), 5, lambda rf: 1),           # odd A, U 0
    "arctic_rf_plus_2000": ((256, 28, 512, 256, 10, 3, 2, 80), 3, lambda rf: rf + 2000),
}
_MODELS = {}


def _dump(name, obj):
    d = os.environ.get("WNB_PARITY_OUT")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, name), "w") as f:
            json.dump(obj, f, indent=1, sort_keys=True)


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 61 + len(_MODELS))).eval()
        net.decode_math = "bf16"
        _MODELS[t] = (cfg, net)
    return _MODELS[t]


def unswizzle(t16, R):
    """queue slots (..., R/64 * 4096) int16 -> (..., 64 rows, R): tile ch // 64 of [64 rows][64 ch] bf16 with the 128B
    swizzle, element (row, ch) at int16 offset (ch // 64) 4096 + 64 row + (((ch % 64) // 8 ^ row) & 7) 8 + ch % 8"""
    KT = R // 64
    t = t16.reshape(*t16.shape[:-1], KT, 64, 8, 8)
    row = torch.arange(64, device=t16.device)
    unit = torch.arange(8, device=t16.device)
    t = t[..., row[:, None], unit[None, :] ^ (row[:, None] & 7), :]       # (..., KT, 64 rows, 8 units, 8)
    return t.movedim(-4, -3).reshape(*t16.shape[:-1], 64, R)


class Queues(object):
    """The decoder's dilation-queue workspace: cluster cl starts at cl q_cluster; layer l's (ks-1) d_l slots start at
    qslot[l] = sum_{k<l} (ks-1) d_k; position t is in slot t mod (ks-1) d_l; row m of cluster cl is utterance
    cl bc + min(m, nu - 1)."""

    def __init__(self, ws, B, R, ks, dil):
        self.B, self.R, self.ks, self.dil = B, R, ks, dil
        self.qlen = [(ks - 1) * d for d in dil]
        self.qslot = np.concatenate([[0], np.cumsum(self.qlen)[:-1]]).astype(int).tolist()
        self.ncl = -(-B // 64)
        self.bc = -(-B // self.ncl)
        self.ws = ws.view(torch.int16).reshape(self.ncl, sum(self.qlen), R * 64)
        self.nu = [min(self.bc, B - cl * self.bc) for cl in range(self.ncl)]

    def rows(self, slots, labels):
        """unswizzled slots (ncl, K, 64, R) -> (B, K, R) bf16, after checking the padding rows (labels[k]: which layer
        and position slot k holds)"""
        for cl, nu in enumerate(self.nu):
            pad = slots[cl, :, nu:, :]
            bad = pad != slots[cl, :, nu - 1:nu, :]
            if bool(bad.any()):
                k, m, c = (int(v) for v in torch.nonzero(bad)[0])
                raise AssertionError("padding row %d of cluster %d differs from its last utterance (row %d) in %s, "
                                     "channel %d: CTA slice %d, 64-channel tile %d (%d values differ)" % (
                                         nu + m, cl, nu - 1, labels[k], c, c // (self.R // 8), c // 64, int(bad.sum())))
        out = torch.cat([slots[cl, :, :nu, :].movedim(1, 0) for cl, nu in enumerate(self.nu)], 0)
        return out.view(torch.bfloat16)

    def history(self, P):
        """every layer's last (ks-1) d_l positions before P - 1: list of (B, qlen_l, R), oldest first"""
        out = []
        for l, ql in enumerate(self.qlen):
            p = np.arange(P - 1 - ql, P - 1)
            idx = torch.as_tensor(self.qslot[l] + p % ql, device=self.ws.device)
            out.append(self.rows(unswizzle(self.ws[:, idx], self.R), ["layer %d position %d" % (l, v) for v in p]))
        return out

    def newest(self, pos):
        """q_l(pos) of every layer: (B, L, R)"""
        idx = torch.as_tensor([self.qslot[l] + pos % ql for l, ql in enumerate(self.qlen)], device=self.ws.device)
        return self.rows(unswizzle(self.ws[:, idx], self.R),
                         ["layer %d position %d" % (l, pos) for l in range(len(self.qlen))])


def _chain(net, x, h, n_list, mode, seed):
    """prefill + one wnb_decode_bf16_at call per position: (codes (B, P + N), logits (B, N, Q) NaN where not written,
    queue history per layer, P)"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import (MODE_ARGMAX, MODE_SAMPLING, _bf16_prefill, _decode_snapshot,
                                                         ptr, stream)
    lib = _lib.load()
    B, T0 = x.shape
    Q, A, Ap, R, S, ks, U, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                                net.upsampling_factor, len(net.dilations))
    P = max(T0, net.receptive_field)
    n_pad, n = P - T0, max(n_list)
    Uc = max(U, 1)
    with torch.no_grad():
        w, upw, upb = _decode_snapshot(net)
        wstream = net._decode_bf16_pack()
    dil = (ctypes.c_int32 * L)(*net.dilations)
    qbytes = lib.wnb_decode_bf16_workspace(B, R, ks, dil, L)
    ws = torch.empty(max(qbytes // 4, 1), dtype=torch.float32, device="cuda")
    codes = torch.full((B, P + n), Q // 2, dtype=torch.int32, device="cuda")
    codes[:, n_pad:P] = x.to(torch.int32)
    _bf16_prefill(lib, codes[:, :P + 1], P, h, upw, upb, w, wstream, dil, L, ws, n_pad, A, Ap, R, S, ks, U)
    qs = Queues(ws, B, R, ks, net.dilations)
    hist = qs.history(P)
    newest = []
    logits = torch.full((B, n, Q), float("nan"), device="cuda")
    cmode = MODE_ARGMAX if mode == "argmax" else MODE_SAMPLING
    for i in range(n):
        pos = P - 1 + i
        if i == 0:   # the first call of a session: xs and h from column 0
            xs_base, hf0 = 0, 0
        else:
            xs_base, hf0 = pos - (ks - 1), max(pos - n_pad, 0) // Uc
        xs = codes[:, xs_base:pos + 2].contiguous()
        hc = h[:, :, hf0:].contiguous()
        nsm = torch.tensor([1 if i < nb else 0 for nb in n_list], dtype=torch.int32, device="cuda")
        lg = torch.full((B, 1, Q), float("nan"), device="cuda")
        _lib.check(lib.wnb_decode_bf16_at(ptr(xs), ptr(hc), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]),
                                          ptr(wstream), dil, L, ptr(ws), ptr(nsm), None, ptr(lg), B, P, 1, n_pad,
                                          hc.size(2), Q, A, Ap, R, S, ks, U, cmode, ctypes.c_uint64(seed), pos, xs_base,
                                          hf0, stream()), "decode_bf16_at")
        codes[:, pos + 1] = xs[:, -1]
        logits[:, i] = lg[:, 0]
        newest.append(qs.newest(pos))
    newest = torch.stack(newest, 1)                                       # (B, N, L, R)
    q = [torch.cat([hist[l], newest[:, :, l]], 1) for l in range(L)]
    q_first = [P - 1 - ql for ql in qs.qlen]
    return codes, logits, q, q_first, P, qs.bc


def _pk(net, n_pad):
    with torch.no_grad():
        wf, bf, W1, b1, W2, b2, Wp1, bp1, Wp2, bp2 = [t.detach().float() for t in net._pack()]
    U = net.upsampling_factor
    return dict(wf=wf, bf=bf, W1=W1, b1=b1, W2=W2, b2=b2, Wp1=Wp1, bp1=bp1, Wp2=Wp2, bp2=bp2,
                up_w=net.upsampling.conv.weight.detach().float().reshape(-1) if U > 0 else None,
                up_b=net.upsampling.conv.bias.detach().float().reshape(-1) if U > 0 else None,
                dil=net.dilations, ks=net.kernel_size, U=U, n_pad=n_pad)


@pytest.mark.parametrize("mode", ["argmax", "philox"])
@pytest.mark.parametrize("case", list(CASES))
def test_bf16_decoder_layers_vs_fp64(case, mode):
    t, B, t0fn = CASES[case]
    cfg, net = _model(t)
    T0 = t0fn(cfg.receptive_field)
    ci = list(CASES).index(case)
    rng = np.random.RandomState(700 + ci)
    U = max(cfg.upsampling_factor, 1)
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T0))).cuda()
    h = torch.from_numpy(rng.standard_normal((B, cfg.n_aux, (T0 + N + U - 1) // U + 1)).astype(np.float32)).cuda()
    n_list = [int(v) for v in rng.randint(1, N + 1, size=B)]
    n_list[0], n_list[1] = 1, N
    bc = -(-B // -(-B // 64))
    for b0 in range(bc, B, bc):      # a cluster whose rows have all finished stops: give each cluster a full-length row
        n_list[b0] = N
    seed = 9000 + ci
    t_start = time.time()
    with torch.no_grad():
        codes, logits, q, q_first, P, bc = _chain(net, x, h, n_list, mode, seed)
        gen, lg1 = net._decode(x, h, n_list, "argmax" if mode == "argmax" else "sampling", return_logits=True,
                               seed=seed)
    assert net.last_decode_kernel == "bf16"
    assert torch.equal(codes[:, P:], gen), "chained codes differ from one-shot decoding"
    for b, nb in enumerate(n_list):
        assert torch.equal(logits[b, :nb], lg1[b, :nb]), ("chained logits differ from one-shot decoding", b)
    rep = DL.check_window(_pk(net, P - T0), codes, h, q, q_first, P - 1, P - 1 + N, logits, bc=bc)
    rep.update(case=case, mode=mode, B=B, L=len(cfg.dilations), P=P, seconds=round(time.time() - t_start, 2))
    _dump("decode_bf16_layers_%s_%s.json" % (case, mode), rep)
    print("bf16 layers %s %s: %s" % (case, mode, rep))
