# -*- coding: utf-8 -*-
"""float64 restatement of held-out scoring (DESIGN.md section 6 row e1), shared by the CPU and GPU tiers: per-row
summed -log softmax(logits)[target] over start <= p < lengths[b], and the number of scored positions."""
import numpy as np


def rows_ce(logits, target, lengths, start):
    """float64 (nll (B,), count (B,)) of (B, T, Q) logits and (B, T) targets: positions start <= p < min(lengths[b],
    T) of row b; a row with none has nll 0 and count 0."""
    B, T, Q = logits.shape
    lg = np.asarray(logits, dtype=np.float64)
    m = lg.max(-1, keepdims=True)
    lse = (m + np.log(np.exp(lg - m).sum(-1, keepdims=True)))[..., 0]
    val = lse - np.take_along_axis(lg, np.asarray(target)[..., None], -1)[..., 0]
    nll, cnt = np.zeros(B), np.zeros(B, dtype=np.int64)
    for b in range(B):
        n = min(int(lengths[b]), T)
        if n > start:
            nll[b], cnt[b] = val[b, start:n].sum(), n - start
    return nll, cnt
