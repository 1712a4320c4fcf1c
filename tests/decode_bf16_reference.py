# -*- coding: utf-8 -*-
"""float64 emulation of the bf16 decoder (csrc/decode_bf16.cu): the teacher-forced forward of tests/decode_reference.py
with the kernel's rounding points.  Every weight except the front embedding is rounded to bf16 (nearest even); every
product's activation operand is rounded to bf16: the aux features, each layer's input (current column and dilated taps),
the gate output z, relu(skip sum) and relu(post-1).  Biases, the residual stream, the skip sum and the nonlinearities
stay float64."""
import numpy as np
import torch

from oracle import wavenet_oracle as O
from tests.decode_reference import _conv


def _bf(t):
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def forward64_bf16(cfg, p, x, h, device="cpu"):
    """x (B, T) int, h (B, A, T) at sample rate -> logits (B, T, Q) float64 numpy, with the bf16 rounding points."""
    def t(k):
        return torch.as_tensor(np.asarray(p[k], np.float64), device=device)

    def w(k):
        return _bf(t(k))

    def b(k):
        return t(k)[None, :, None]

    W = t("causal.conv.weight")
    R, Q, ks = W.shape
    x = torch.as_tensor(np.asarray(x, np.int64), device=device) % Q
    h = _bf(torch.as_tensor(np.asarray(h, np.float64), device=device))
    B, T = x.shape
    out = b("causal.conv.bias").expand(B, R, T).clone()
    for k in range(ks):
        s = ks - 1 - k
        if s < T:
            out[:, :, s:] += W[:, :, k].t()[x[:, :T - s]].transpose(1, 2)
    skip = 0
    for l, d in enumerate(cfg.dilations):
        xb = _bf(out)
        a = _conv(w("dil_sigmoid.%d.conv.weight" % l), xb, d) + b("dil_sigmoid.%d.conv.bias" % l) + \
            _conv(w("aux_1x1_sigmoid.%d.weight" % l), h) + b("aux_1x1_sigmoid.%d.bias" % l)
        g = _conv(w("dil_tanh.%d.conv.weight" % l), xb, d) + b("dil_tanh.%d.conv.bias" % l) + \
            _conv(w("aux_1x1_tanh.%d.weight" % l), h) + b("aux_1x1_tanh.%d.bias" % l)
        z = _bf(torch.sigmoid(a) * torch.tanh(g))
        skip = skip + _conv(w("skip_1x1.%d.weight" % l), z) + b("skip_1x1.%d.bias" % l)
        out = _conv(w("res_1x1.%d.weight" % l), z) + b("res_1x1.%d.bias" % l) + out
    r1 = _bf(torch.relu(_conv(w("conv_post_1.weight"), _bf(torch.relu(skip))) + b("conv_post_1.bias")))
    y = _conv(w("conv_post_2.weight"), r1) + b("conv_post_2.bias")
    return y.transpose(1, 2).cpu().numpy()


def teacher_forced_logits_bf16(cfg, p64, x, h, samples, device="cuda", chunk=8):
    """``decode_reference.teacher_forced_logits`` with ``forward64_bf16`` in place of the float64 forward."""
    xp, hp = O._pad_inputs(cfg, p64, np.asarray(x, np.int64), np.asarray(h, np.float64))
    P = xp.shape[1]
    samples = np.asarray(samples, np.int64)
    n = samples.shape[1]
    seq = np.concatenate([xp, samples[:, :n - 1]], 1)
    hs = hp[:, :, :P - 1 + n]
    c0 = O.Config(*cfg.as_tuple()[:7] + (0,))
    B = seq.shape[0]
    return np.concatenate([forward64_bf16(c0, p64, seq[i:i + chunk], hs[i:i + chunk], device)[:, P - 1:P - 1 + n]
                           for i in range(0, B, chunk)], 0)
