# -*- coding: utf-8 -*-
"""GPU tier: the BENCHMARKED paths compared DIRECTLY with the float64 oracle (no CUDA-vs-CUDA links).

* tf32 deferred-skip stack (csrc/stack.cu, the bench path) at the BASELINE configs[1] architecture
  ``WaveNet(256,28,64,512,10,3,2,80)``, B=2, T=4160 (time tiles well past the receptive field 3070): loss and
  EVERY parameter gradient vs ``oracle.backward`` in float64 (reference bin/train.py:530-538 over
  nets/wavenet.py:212-241).  The observed error of every tensor is printed (and written as parity_*.json into the
  directory named by $WNB_PARITY_OUT, when set) so that the asserted tolerances are the measured ones x ~2, not a guess.
* the composed tensor-core path at the ljspeech-melspc architecture ``(256,80,512,256,10,3,3,256)`` on a short window
  (reference egs/ljspeech/sd-melspc/run.sh:28-33).
* long free-running argmax decode (>= 10 000 samples, all three kernels) vs ``oracle.batch_fast_generate`` with the
  first-divergence / top-2-margin protocol of SURVEY.md 8c-4(iii) (reference nets/wavenet.py:309-395).
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

def _dump(name, obj):
    d = os.environ.get("WNB_PARITY_OUT")
    if not d:
        return
    try:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, name), "w") as f:
            json.dump(obj, f, indent=1, sort_keys=True)
    except OSError:
        pass


def _grad_errors(net, gref):
    """per tensor: relative Frobenius error and max-abs error relative to max|ref|"""
    rows = {}
    for k, prm in net.named_parameters():
        ref = gref[k]
        if prm.grad is None:
            rows[k] = None
            continue
        got = prm.grad.detach().cpu().numpy().astype(np.float64).reshape(ref.shape)
        nref = float(np.linalg.norm(ref))
        rows[k] = {"rel_fro": float(np.linalg.norm(got - ref) / max(nref, 1e-30)),
                   "max_abs_over_max_ref": float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)),
                   "ref_norm": nref, "numel": int(ref.size)}
    return rows


def _train_step_vs_oracle(cfg, seed, B, T, start, math_mode, expect_stack):
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    p = O.make_params(cfg, seed)
    net = our_model(cfg, p, math_mode=math_mode).train()
    lib = _lib.load()
    if expect_stack is not None:
        sup = bool(lib.wnb_stack_supported(cfg.n_resch, cfg.n_skipch, net.n_aux_pad, cfg.kernel_size,
                                           len(cfg.dilations), net._math()))
        assert sup == expect_stack
    net._wnb_debug = {}
    rng = np.random.RandomState(seed + 100)
    U = max(cfg.upsampling_factor, 1)
    x = rng.randint(0, cfg.n_quantize, size=(B, T)).astype(np.int64)
    t = rng.randint(0, cfg.n_quantize, size=(B, T)).astype(np.int64)
    h = rng.standard_normal((B, cfg.n_aux, T // U)).astype(np.float32)
    y = net(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda())
    loss = cross_entropy(y, torch.from_numpy(t).cuda(), start)
    loss.backward()
    torch.cuda.synchronize()
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    ref, cache = O.forward(cfg, p64, x, h.astype(np.float64), return_cache=True)
    rl, dl = O.cross_entropy(ref, t, start)
    g = O.backward(cfg, p64, cache, dl)
    yv = y.detach().cpu().numpy().astype(np.float64)
    rows = _grad_errors(net, g)
    rows_same_masks, flips = None, None
    if "skip_mask" in net._wnb_debug:
        # the same comparison with the oracle's two post-network ReLU masks replaced by the sign patterns of OUR forward:
        # isolates the arithmetic error of the backward kernels from mask flips at pre-activations within rounding
        # distance of zero (each flip passes / blocks a whole gradient element)
        ms = net._wnb_debug["skip_mask"].cpu().numpy().transpose(0, 2, 1)
        m1 = net._wnb_debug["r1_mask"].cpu().numpy().transpose(0, 2, 1)
        flips = {"skip": float((ms != (cache["skip_sum"] > 0))[:, :, start:].mean()),
                 "h1": float((m1 != (cache["post"][1] > 0))[:, :, start:].mean())}
        rows_same_masks = _grad_errors(net, O.backward(cfg, p64, cache, dl, relu_masks={"h1": m1, "skip": ms}))
    srt = np.sort(ref, axis=-1)
    margin = srt[..., -1] - srt[..., -2]
    agree = (yv.argmax(-1) == ref.argmax(-1))
    rep = {"cfg": list(cfg.as_tuple()), "B": B, "T": T, "loss_start": start, "math": math_mode,
           "loss": float(loss.item()), "loss_oracle": float(rl), "loss_abs_err": abs(float(loss.item()) - float(rl)),
           "logits_max_abs_err": float(np.abs(yv - ref).max()), "logits_max_ref": float(np.abs(ref).max()),
           "argmax_agree_all": float(agree.mean()),
           "argmax_agree_margin_gt_0.05": float(agree[margin > 0.05].mean()) if (margin > 0.05).any() else None,
           "grads": rows, "grads_same_relu_masks": rows_same_masks, "relu_mask_flip_fraction": flips}
    return rep


def _worst(rows, pred):
    sel = {k: v for k, v in rows.items() if v is not None and pred(k, v)}
    k = max(sel, key=lambda kk: sel[kk]["rel_fro"])
    return k, sel[k]["rel_fro"]


def _is_weight(k, v):
    return k.endswith("weight") and v["numel"] > 1


def _is_bias(k, v):
    return k.endswith("bias") and v["numel"] > 1


def _summarise(rep):
    rows = rep["grads"]
    rep["worst_weight"] = _worst(rows, _is_weight)
    rep["worst_bias"] = _worst(rows, _is_bias)
    if rep.get("grads_same_relu_masks"):
        rep["worst_weight_same_masks"] = _worst(rep["grads_same_relu_masks"], _is_weight)
        rep["worst_bias_same_masks"] = _worst(rep["grads_same_relu_masks"], _is_bias)
    per_kind = {}
    for k, v in rows.items():
        if v is None:
            continue
        kind = ".".join(s for s in k.split(".") if not s.isdigit())
        per_kind.setdefault(kind, []).append(v["rel_fro"])
    rep["rel_fro_by_kind"] = {k: {"max": max(v), "median": float(np.median(v))} for k, v in per_kind.items()}
    return rep


def test_tf32_stack_every_gradient_vs_fp64_oracle_arctic30():
    """The bench path: 30 blocks, 64 res / 512 skip, kernel 2, U = 80; all 184 gradient tensors vs the fp64 oracle.

    Tolerances (asserted) = about twice the error observed (see the note above TOL_TF32):
    tf32 rounds both operands of every contraction to 10 mantissa bits (2^-11 relative), the gate uses
    tanh.approx.f32 (2^-10.987 max relative error); the gradients at the bottom of the stack carry the rounding of
    every block above them."""
    cfg = O.Config(256, 28, 64, 512, 10, 3, 2, 80)
    rep = _summarise(_train_step_vs_oracle(cfg, 3, 2, 4160, cfg.receptive_field, "tf32", True))
    _dump("parity_stack_arctic_tf32.json", rep)
    print("tf32 stack vs fp64 oracle: loss err %.2e, logits max err %.2e, worst weight %s %.3e, worst bias %s %.3e"
          % (rep["loss_abs_err"], rep["logits_max_abs_err"], rep["worst_weight"][0], rep["worst_weight"][1],
             rep["worst_bias"][0], rep["worst_bias"][1]))
    print("   with the oracle's ReLU masks replaced by ours (flip fraction %s): worst weight %s %.3e, worst bias %s %.3e"
          % (rep["relu_mask_flip_fraction"], rep["worst_weight_same_masks"][0], rep["worst_weight_same_masks"][1],
             rep["worst_bias_same_masks"][0], rep["worst_bias_same_masks"][1]))
    assert rep["loss_abs_err"] < TOL_TF32["loss"], rep["loss_abs_err"]
    assert rep["logits_max_abs_err"] < TOL_TF32["logits"], rep["logits_max_abs_err"]
    none = [k for k, v in rep["grads"].items() if v is None]
    assert none == ["res_1x1.29.weight", "res_1x1.29.bias"], none   # reference: the last res_1x1 gets no gradient
    for key, tols in (("grads", TOL_TF32), ("grads_same_relu_masks", TOL_TF32_SAME_MASKS)):
        for k, v in rep[key].items():
            if v is None:
                continue
            if v["numel"] == 1:     # upsampling bias: one scalar = a sum with heavy cancellation, no relative bound
                continue
            tol = tols["weight"] if k.endswith("weight") else tols["bias"]
            assert v["rel_fro"] <= tol, (key, k, v)


def test_fp32_path_every_gradient_vs_fp64_oracle_arctic30():
    """Same comparison for math_mode="fp32" (FFMA kernels): the parity path, errors at fp32 rounding level."""
    cfg = O.Config(256, 28, 64, 512, 10, 3, 2, 80)
    rep = _summarise(_train_step_vs_oracle(cfg, 3, 2, 4160, cfg.receptive_field, "fp32", None))
    _dump("parity_stack_arctic_fp32.json", rep)
    print("fp32 path vs fp64 oracle: loss err %.2e, logits max err %.2e, worst weight %s %.3e, worst bias %s %.3e"
          % (rep["loss_abs_err"], rep["logits_max_abs_err"], rep["worst_weight"][0], rep["worst_weight"][1],
             rep["worst_bias"][0], rep["worst_bias"][1]))
    assert rep["loss_abs_err"] < 1e-5
    assert rep["logits_max_abs_err"] < 1e-4
    for k, v in rep["grads"].items():
        if v is None or v["numel"] == 1:
            continue
        assert v["rel_fro"] <= 1e-3, (k, v)


def test_composed_tf32_path_vs_fp64_oracle_ljspeech_melspc():
    """configs[2] architecture (512 res / 256 skip, kernel 3, 80-dim mel aux, U = 256) on a short window: the
    composed tensor-core path (per-block GEMMs) vs the fp64 oracle, loss + every gradient."""
    cfg = O.Config(256, 80, 512, 256, 10, 3, 3, 256)
    rep = _summarise(_train_step_vs_oracle(cfg, 5, 1, 768, 128, "tf32", False))
    _dump("parity_composed_ljspeech_tf32.json", rep)
    print("composed tf32 vs fp64 oracle: loss err %.2e, logits max err %.2e, worst weight %s %.3e, worst bias %s %.3e"
          % (rep["loss_abs_err"], rep["logits_max_abs_err"], rep["worst_weight"][0], rep["worst_weight"][1],
             rep["worst_bias"][0], rep["worst_bias"][1]))
    assert rep["loss_abs_err"] < TOL_COMPOSED["loss"]
    assert rep["logits_max_abs_err"] < TOL_COMPOSED["logits"]
    for k, v in rep["grads"].items():
        if v is None or v["numel"] == 1:
            continue
        tol = TOL_COMPOSED["weight"] if k.endswith("weight") else TOL_COMPOSED["bias"]
        assert v["rel_fro"] <= tol, (k, v)


# Asserted tolerances: ~2x the errors observed.  Observed on an H100: loss 1.1e-3, logits 1.4e-2 (max |logit| 3.2),
# weight gradients up to 5.7 %, biases up to 6.5 % -- already 2.5 % at conv_post_1: it is not rounding accumulated through
# the stack but the two ReLU masks of the post network flipping where a pre-activation is within tf32 rounding of zero.
# With the masks shared the same gradients agree to the second set of bounds.
TOL_TF32 = {"loss": 2.5e-3, "logits": 3e-2, "weight": 0.08, "bias": 0.09}
# observed with shared masks: weights 0.35-0.90 % (tf32 rounding accumulated through the stack), biases <= 0.85 %; mask
# flip fraction 7e-4 per ReLU
TOL_TF32_SAME_MASKS = {"weight": 0.018, "bias": 0.018}
# composed path at the ljspeech-melspc shape (observed: loss 5.1e-3, logits 2.4e-2 at max |logit| 5.3, weights <= 5.2 %,
# biases <= 2.8 %; the same ReLU-mask effect, K = 512..1616 contractions)
TOL_COMPOSED = {"loss": 1e-2, "logits": 5e-2, "weight": 0.08, "bias": 0.05}


@pytest.mark.parametrize("kernel", ["warp", "stream", "direct"])
def test_decode_long_run_first_divergence_protocol(kernel):
    """SURVEY.md 8c-4(iii): >= 10 000 free-running argmax samples per utterance at the BASELINE decode architecture
    vs the float64 oracle.  Either the index sequences are identical, or at the FIRST differing position the oracle's
    top-2 logit margin is below 1e-5 (an fp32-rounding tie; the trajectories are incomparable afterwards)."""
    cfg = O.Config(256, 28, 64, 512, 10, 3, 2, 80)
    p = O.make_params(cfg, 11)
    net = our_model(cfg, p).eval()
    rng = np.random.RandomState(13)
    B, n = 3, 10000
    frames = (n + 1 + 79) // 80
    x = np.full((B, 1), 128, np.int64)
    h = rng.standard_normal((B, 28, frames)).astype(np.float32)
    with torch.no_grad():
        gen = net._decode(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), [n] * B, "argmax", kernel=kernel)
    assert net.last_decode_kernel == kernel
    gen = gen.cpu().numpy()
    ref = _oracle_long_run(cfg, p, x, h, n)
    rep = []
    for b in range(B):
        diff = np.nonzero(gen[b, :n] != ref["samples"][b])[0]
        if diff.size == 0:
            rep.append({"utt": b, "identical": True, "samples": n, "min_margin_seen": float(ref["margin"][b].min())})
            continue
        i = int(diff[0])
        rep.append({"utt": b, "identical": False, "first_divergence": i, "oracle_margin_there": float(ref["margin"][b, i]),
                    "ours": int(gen[b, i]), "oracle": int(ref["samples"][b, i]),
                    "oracle_top2": [int(v) for v in ref["top2"][b, i]]})
    _dump("decode_long_run_%s.json" % kernel, rep)
    print("decode long run (%s): %s" % (kernel, rep))
    for r in rep:
        if not r["identical"]:
            assert r["oracle_margin_there"] < 1e-5, r
            assert r["ours"] in r["oracle_top2"], r


_LONG_RUN_CACHE = {}


def _oracle_long_run(cfg, p, x, h, n):
    """float64 oracle trajectory + per-step top-2 margin (computed once per session, shared by the three kernels)."""
    key = (n, x.shape[0])
    if key not in _LONG_RUN_CACHE:
        p64 = {k: v.astype(np.float64) for k, v in p.items()}
        outs, lg = O.batch_fast_generate(cfg, p64, x, h.astype(np.float64), [n] * x.shape[0], mode="argmax",
                                         return_logits=True)
        srt = np.argsort(lg, axis=-1)
        top2 = srt[..., -2:][..., ::-1]
        s = np.sort(lg, axis=-1)
        _LONG_RUN_CACHE[key] = {"samples": np.stack(outs), "margin": s[..., -1] - s[..., -2], "top2": top2}
    return _LONG_RUN_CACHE[key]
