# -*- coding: utf-8 -*-
"""Held-out scoring: the teacher-forced negative log-likelihood of utterances given their features (DESIGN.md
section 6, row e1), which is the training loss computed on audio the model has not seen.

Each utterance is aligned exactly as the training batches are (``bin/train.py`` ``train_generator``):
``utterance_arrays`` gives its inputs (mu-law codes without the last sample), targets (the codes from the second
sample) and aux features.  ``score_utterances`` batches a list under a sample budget, runs ``WaveNet.score`` and
returns, per utterance and in list order, the summed NLL in nats and the number of scored positions.  The corpus
figure is ``corpus_mean``: the sums added in list order over the counts added in list order.

An utterance too long for the budget is scored in windows (``score_window_plan``).  Each window repeats enough
context before the positions it scores that they see exactly the inputs they see in the whole utterance, and the
windows are chained through ``WaveNet.score(out=...)``, so the result equals whole-utterance scoring bit for bit
wherever the forward computes each position the same way in both (DESIGN.md section 6).
"""
import math

import numpy as np
import torch

# the column segment of wnb_cross_entropy_rows (csrc/score.cu): window starts must be multiples of it
SEGMENT = 32


def window_unit(upsampling_factor):
    """Windows start, and hop, at multiples of this many samples: whole frames of the up-sampling layer (U > 0) and
    whole summation segments of the scoring kernel."""
    U = int(upsampling_factor)
    return SEGMENT * U // math.gcd(SEGMENT, U) if U > 0 else SEGMENT


def window_context(receptive_field, upsampling_factor):
    """Samples a window repeats before the first position it scores: ``receptive_field - 1`` rounded up to
    ``window_unit``, so that every scored position sees no zero padding the whole utterance does not also see."""
    unit = window_unit(upsampling_factor)
    return (receptive_field - 1 + unit - 1) // unit * unit


def score_window_plan(T, receptive_field, upsampling_factor, L, start):
    """Windows that score positions ``start <= p < T`` of one utterance, each exactly once.

    ``L`` (a positive multiple of ``window_unit``) is the hop.  Window k scores ``[max(start, k L), min((k + 1) L, T))``
    and reads inputs ``[max(0, k L - C), min((k + 1) L, T))`` with C = ``window_context``: at most C + L positions, of
    which the last L (fewer in the first and last windows) are scored.  Returns ``[(k, a, s, e)]``: input start a,
    scored range [s, e), windows with nothing to score left out."""
    unit = window_unit(upsampling_factor)
    if L <= 0 or L % unit:
        raise ValueError("window hop %d should be a positive multiple of %d" % (L, unit))
    if start < 0:
        raise ValueError("start should be >= 0, got %d" % start)
    C = window_context(receptive_field, upsampling_factor)
    plan = []
    for k in range(start // L, (T + L - 1) // L):
        s, e = max(start, k * L), min((k + 1) * L, T)
        if s < e:
            plan.append((k, max(0, k * L - C), s, e))
    return plan


def utterance_arrays(x, h, n_quantize, upsampling_factor, mulaw=None):
    """One utterance aligned as ``train_generator`` aligns it: ``(x_in (T,) int64, t (T,) int64, h float32)``.

    ``x`` is the waveform and ``h`` the scaled (frames, D) features after ``validate_length`` (``bin/train.py``
    ``_load_pair``).  With an up-sampling layer (U > 0) F' = min(frames, (len(x) - 1) // U) frames and T = F' U
    samples are used, h is (D, F'); without one h is already at the sample rate and is (D, T) with T = len(x) - 1.
    x_in = mu-law(x)[:T] and t = mu-law(x)[1:T + 1], with ``mulaw`` (default ``nets.encode_mu_law``, on the GPU)."""
    if mulaw is None:
        from pytorchwavenetvocoder_b200.nets import encode_mu_law as mulaw
    U = int(upsampling_factor)
    x = np.asarray(x)
    h = np.asarray(h, dtype=np.float32)
    if U > 0:
        F = max(0, min(h.shape[0], (len(x) - 1) // U))
        T = F * U
        hh = h[:F]
    else:
        T = max(0, min(len(x), h.shape[0]) - 1)
        hh = h[:T]
    codes = np.asarray(mulaw(x[:T + 1], n_quantize), dtype=np.int64)
    return codes[:T], codes[1:T + 1], np.ascontiguousarray(hh.T)


def load_utterance(wavfile, featfile, config, scaler):
    """``utterance_arrays`` of one (wav, feat) pair under ``config`` (model.conf), features scaled by ``scaler``."""
    from pytorchwavenetvocoder_b200.bin.train import _load_pair
    x, h = _load_pair(wavfile, featfile, config.feature_type, config.upsampling_factor, config.use_upsampling_layer,
                      config.use_speaker_code)
    U = config.upsampling_factor if config.use_upsampling_layer else 0
    return utterance_arrays(x, scaler.transform(h), config.n_quantize, U)


def score_batches(lengths, batch_samples):
    """Batches of utterance indices for ``score_utterances``: longest first, each batch's rows x longest length within
    ``batch_samples``.  An utterance longer than the budget is a batch of its own (scored in windows)."""
    order = sorted(range(len(lengths)), key=lambda i: (-lengths[i], i))
    batches, cur = [], []
    for i in order:
        if cur and (len(cur) + 1) * lengths[cur[0]] > batch_samples:
            batches.append(cur)
            cur = []
        cur.append(i)
    if cur:
        batches.append(cur)
    return batches


def _upload(rows, T, U, n_aux, device="cuda"):
    """Zero-padded (B, T) inputs and targets and (B, D, T or T / U) aux of ``rows`` = [(x_in, t, h)] on ``device``."""
    B = len(rows)
    xb = np.zeros((B, T), dtype=np.int64)
    tb = np.zeros((B, T), dtype=np.int64)
    hb = np.zeros((B, n_aux, T // U if U > 0 else T), dtype=np.float32)
    for b, (x, t, h) in enumerate(rows):
        xb[b, :len(x)], tb[b, :len(t)], hb[b, :, :h.shape[1]] = x, t, h
    return tuple(torch.from_numpy(v).to(device) for v in (xb, tb, hb))


def score_windows(model, utts, L, start, out):
    """Score ``utts`` = [(x_in, t, h)] (longest first) in windows of hop ``L`` (``score_window_plan``), adding into
    ``out`` = (nll (B,), count (B,)) on the device.  Window k of every utterance that has one runs in one
    ``WaveNet.score`` call; those utterances are a prefix of the list, so the call adds into a prefix of ``out``."""
    U, rf = model.upsampling_factor, model.receptive_field
    dev = out[0].device
    Tmax = len(utts[0][0])
    for k, a, s, e in score_window_plan(Tmax, rf, U, L, start):
        rows = []
        for x, t, h in utts:
            e_b = min(e, len(x))
            if e_b <= s:
                break
            f0, f1 = (a // U, e_b // U) if U > 0 else (a, e_b)
            rows.append((x[a:e_b], t[a:e_b], h[:, f0:f1]))
        xb, tb, hb = _upload(rows, e - a, U, model.n_aux, dev)
        lengths = torch.tensor([len(r[0]) for r in rows], dtype=torch.int64).to(dev)
        n = len(rows)
        model.score(xb, hb, tb, lengths, s - a, out=(out[0][:n], out[1][:n]))


def score_utterances(model, utts, batch_samples, start=None):
    """Per-utterance ``(nll float64 (N,), count int64 (N,))`` numpy arrays, in the order of ``utts`` = [(x_in, t, h)]
    (``utterance_arrays``).  Batches follow ``score_batches``; an utterance longer than ``batch_samples`` is scored
    alone in windows whose hop is the largest multiple of ``window_unit`` that keeps a window within the budget."""
    start = model.receptive_field if start is None else int(start)
    N = len(utts)
    nll, count = np.zeros(N, dtype=np.float64), np.zeros(N, dtype=np.int64)
    lengths = [len(u[0]) for u in utts]
    live = [i for i in range(N) if lengths[i] > start]   # nothing to score: count 0, nll 0, no forward
    U = model.upsampling_factor
    dev = next(model.parameters()).device
    results = []
    for batch in score_batches([lengths[i] for i in live], batch_samples):
        idx = [live[j] for j in batch]
        rows = [utts[i] for i in idx]
        T = lengths[idx[0]]
        if T <= batch_samples:
            xb, tb, hb = _upload(rows, T, U, model.n_aux, dev)
            results.append((idx, model.score(xb, hb, tb, [lengths[i] for i in idx], start)))
            continue
        unit = window_unit(U)
        C = window_context(model.receptive_field, U)
        L = max(unit, (batch_samples - C) // unit * unit)
        out = (torch.zeros(len(rows), dtype=torch.float64, device=dev),
               torch.zeros(len(rows), dtype=torch.int64, device=dev))
        score_windows(model, rows, L, start, out)
        results.append((idx, out))
    for idx, (n_, c_) in results:
        nll[idx], count[idx] = n_.cpu().numpy(), c_.cpu().numpy()
    return nll, count


def corpus_mean(nll, count):
    """(Σ nll, Σ count, Σ nll / Σ count) with both sums taken in list order; the mean is NaN when nothing was
    scored.  Utterances with count 0 add nothing."""
    s, n = 0.0, 0
    for v, c in zip(nll, count):
        s += float(v)
        n += int(c)
    return s, n, (s / n if n > 0 else float("nan"))

