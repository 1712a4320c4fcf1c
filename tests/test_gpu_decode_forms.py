# -*- coding: utf-8 -*-
"""GPU tier: every launch form of the three decode kernels, step by step against float64.

* all eight ``decode_warp_kernel<NU, W, BIG, CL>`` instantiations, each reached on purpose (B from the device's SM
  count, WNB_DECODE_BIG=0 for the small-slot forms, L <= 9 for <4,8,true,1>) and checked through
  ``wnb_decode_warp_form``, plus the speaker-code shape (U = 0, A = 31), A = 32 and WNB_DECODE_SPLIT=8;
* the streaming and direct kernels with 1, 2 and 4 utterances per CTA, and at the recipes' 512/256 sizes at full
  dilation range (queues of up to 2 x 512 slots that wrap);
* 10 000-step runs in sampling mode with in-kernel Philox (the bench's mode) on the cluster and single-CTA warp forms,
  the streaming and the direct kernel: the error must not grow with time;
* a CDF-boundary sweep: uniforms that put the sampling target within +-8 ulps of every lane boundary, for these forms
  and for the bf16 decoder's own pick.

Every case gives each utterance its own multi-sample seed and aux, ragged lengths (1 and max_n among them, different
inside one CTA) and a batch that is not a multiple of the utterances per CTA.  Every step's logits are compared with
the teacher-forced float64 forward (tests/decode_reference.py), every pick is checked (first maximum for argmax; inside
the admissible set of the kernel's own logits for sampling, with ``philox_uniform`` when the kernel draws), and
``gen[b, n_b:]`` must still hold Q // 2.  Observed errors are printed and, when $WNB_PARITY_OUT is set, written there as
decode_forms_*.json; the asserted bounds are about twice the largest observed on an H100 (see TOL_*).
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests import decode_reference as D
from tests.util import our_model

pytestmark = pytest.mark.gpu

# Asserted bounds on |logit - float64|, about twice the worst observed on an H100 80GB HBM3 (DESIGN.md section 4):
TOL_64 = 5e-6        # 64 res / 512 skip: observed <= 2.1e-6 over all forms, modes and the 10 000-step runs
TOL_512 = 2e-5       # the recipes' 512 res / 256 skip: observed <= 8.2e-6
SHALLOW = (256, 28, 64, 512, 4, 2, 2, 4)      # L = 8: keeps the oracle cheap at B ~ 270
BENCH = (256, 28, 64, 512, 10, 3, 2, 80)      # L = 30: the bench's decode shape


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


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


_MODELS = {}


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        p = O.make_params(cfg, 17 + len(_MODELS))
        _MODELS[t] = (cfg, our_model(cfg, p).eval(), {k: v.astype(np.float64) for k, v in p.items()})
    return _MODELS[t]


def _warp_form(B, L):
    from pytorchwavenetvocoder_b200 import _lib
    f = (ctypes.c_int32 * 4)()
    _lib.check(_lib.load().wnb_decode_warp_form(B, L, f), "decode_warp_form")
    return tuple(int(v) for v in f)


def _inputs(cfg, B, T0, max_n, seed):
    """per-utterance seeds and aux; ragged lengths with 1 and max_n in the first CTA"""
    rng = np.random.RandomState(seed)
    U = max(cfg.upsampling_factor, 1)
    x = rng.randint(0, cfg.n_quantize, size=(B, T0)).astype(np.int64)
    h = rng.standard_normal((B, cfg.n_aux, (T0 + max_n + U - 1) // U + 1)).astype(np.float32)
    n_list = [int(v) for v in rng.randint(1, max_n + 1, size=B)]
    n_list[0] = 1
    if B > 1:
        n_list[1] = max_n
    return x, h, n_list


def _decode(net, x, h, n_list, mode, kernel, uniforms=None, seed=None, expect=None):
    """decode with ``kernel`` and check that ``expect`` (default: the kernel named) ran"""
    with torch.no_grad():
        gen, lg = net._decode(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), n_list, mode,
                              uniforms=None if uniforms is None else torch.from_numpy(uniforms),
                              return_logits=True, seed=seed, kernel=kernel)
    assert net.last_decode_kernel == (expect or kernel), (kernel, net.last_decode_kernel)
    return gen.cpu().numpy().astype(np.int64), lg.cpu().numpy()


def _check(cfg, p64, x, h, n_list, gen, lg, mode, uni, refs=None):
    """per-step logit errors vs the teacher-forced float64 forward and every pick; returns (errors (B, max_n) with NaN
    past n_b, list of bad picks).  A dict ``refs`` receives the float64 logits as ``refs["ref"]``."""
    B, max_n = len(n_list), max(n_list)
    Q = cfg.n_quantize
    ref = D.teacher_forced_logits(cfg, p64, x, h, gen[:, :max_n], device="cuda", chunk=8)
    if refs is not None:
        refs["ref"] = ref
    err = np.full((B, max_n), np.nan)
    bad = []
    for b in range(B):
        nb = n_list[b]
        assert np.all(gen[b, nb:] == Q // 2), ("samples written past n_b", b, nb)
        err[b, :nb] = np.abs(lg[b, :nb].astype(np.float64) - ref[b, :nb]).max(-1)
        picks = gen[b, :nb]
        if mode == "argmax":
            ok = picks == np.argmax(lg[b, :nb], -1)
        else:
            ok = D.admissible(lg[b, :nb], uni[b, :nb])[np.arange(nb), picks]
        for i in np.nonzero(~ok)[0][:5]:
            bad.append({"utt": b, "step": int(i), "pick": int(picks[i]),
                        "uni": None if uni is None else float(uni[b, i])})
    return err, bad


def _run_modes(cfg, net, p64, x, h, n_list, kernel, seed, expect=None, on_mode=None):
    """argmax, sampling with supplied uniforms and sampling with in-kernel Philox: worst logit error per mode.
    ``on_mode(mode, gen, lg, ref)``, when given, returns a dict of further results for the mode's row."""
    rng = np.random.RandomState(seed)
    B, max_n = len(n_list), max(n_list)
    rows = {}
    for mode in ("argmax", "uniforms", "philox"):
        uni = None
        if mode == "uniforms":
            uni = rng.uniform(size=(B, max_n)).astype(np.float32)
            gen, lg = _decode(net, x, h, n_list, "sampling", kernel, uniforms=uni, expect=expect)
        elif mode == "philox":
            gen, lg = _decode(net, x, h, n_list, "sampling", kernel, seed=seed, expect=expect)
            uni = D.philox_uniform(seed, np.arange(B)[:, None], np.arange(max_n)[None, :])
        else:
            gen, lg = _decode(net, x, h, n_list, "argmax", kernel, expect=expect)
        refs = {}
        err, bad = _check(cfg, p64, x, h, n_list, gen, lg, "argmax" if mode == "argmax" else "sampling", uni, refs)
        rows[mode] = {"max_err": float(np.nanmax(err)), "bad_picks": bad,
                      "max_abs_logit": float(np.abs(lg[0, :n_list[0]]).max())}
        if on_mode is not None:
            rows[mode].update(on_mode(mode, gen, lg, refs["ref"]))
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# the eight warp-tiled forms (+ three shapes on the cluster form)
# ---------------------------------------------------------------------------------------------------------------------
# id -> (cfg, B as a function of the SM count, WNB_DECODE_BIG, WNB_DECODE_SPLIT, expected (NU, W, CL, BIG))
WARP_FORMS = {
    "1x16_big_cl2": (BENCH, lambda n: n // 2 - 1, None, None, (1, 16, 2, 1)),
    "1x16_big_cl1": (BENCH, lambda n: n // 2 + 3, None, None, (1, 16, 1, 1)),
    "1x16_small_cl2": (SHALLOW, lambda n: n // 2 - 1, "0", None, (1, 16, 2, 0)),
    "1x16_small_cl1": (SHALLOW, lambda n: n - 1, "0", None, (1, 16, 1, 0)),
    "2x16_big": (SHALLOW, lambda n: n + 7, None, None, (2, 16, 1, 1)),
    "2x16_small": (SHALLOW, lambda n: 2 * n - 1, "0", None, (2, 16, 1, 0)),
    "4x8_big": ((256, 28, 64, 512, 3, 3, 2, 4), lambda n: 2 * n + 7, None, None, (4, 8, 1, 1)),   # L = 9
    "4x8_small": ((256, 28, 64, 512, 6, 2, 2, 4), lambda n: 2 * n + 9, None, None, (4, 8, 1, 0)),  # L = 12
    "speaker_A31_U0": ((256, 31, 64, 512, 4, 2, 2, 0), lambda n: 5, None, None, (1, 16, 2, 1)),
    "A32": ((256, 32, 64, 512, 4, 2, 2, 4), lambda n: 5, None, None, (1, 16, 2, 1)),
    "split8": (SHALLOW, lambda n: 7, None, "8", (1, 16, 2, 1)),
}


def _setup_warp(form_id, monkeypatch):
    t, bfn, big, split, want = WARP_FORMS[form_id]
    if big is not None:
        monkeypatch.setenv("WNB_DECODE_BIG", big)
    if split is not None:
        monkeypatch.setenv("WNB_DECODE_SPLIT", split)
    cfg, net, p64 = _model(t)
    B = bfn(_nsm())
    got = _warp_form(B, len(cfg.dilations))
    assert got == want, (form_id, B, got)
    assert B % want[0] != 0 or want[0] == 1
    return cfg, net, p64, B, got


@pytest.mark.parametrize("form_id", list(WARP_FORMS))
def test_warp_form_vs_fp64(form_id, monkeypatch):
    cfg, net, p64, B, form = _setup_warp(form_id, monkeypatch)
    ci = list(WARP_FORMS).index(form_id)
    T0 = 5 if ci % 2 == 0 else cfg.receptive_field + 9
    x, h, n_list = _inputs(cfg, B, T0, 32, 100 + ci)
    rows = _run_modes(cfg, net, p64, x, h, n_list, "warp", 1000 + ci)
    rep = {"form (NU, W, CL, BIG)": form, "B": B, "L": len(cfg.dilations), "T0": T0, "modes": rows, "tol": TOL_64}
    _dump("decode_forms_warp_%s.json" % form_id, rep)
    print("warp %s: form %s B=%d L=%d: max logit err %s (tol %.1e)" % (
        form_id, form, B, len(cfg.dilations), {m: "%.2e" % r["max_err"] for m, r in rows.items()}, TOL_64))
    for m, r in rows.items():
        assert not r["bad_picks"], (m, r["bad_picks"])
        assert r["max_err"] <= TOL_64, (m, r["max_err"])


# ---------------------------------------------------------------------------------------------------------------------
# streaming and direct kernels: 1 / 2 / 4 utterances per CTA, and the recipe sizes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["stream", "direct"])
@pytest.mark.parametrize("nu", [1, 2, 4])
def test_stream_direct_nu_vs_fp64(kernel, nu):
    cfg, net, p64 = _model(SHALLOW)
    nsm = _nsm()
    B = {1: 5, 2: nsm + 5, 4: 2 * nsm + 5}[nu]
    x, h, n_list = _inputs(cfg, B, 4 if nu != 2 else 40, 32, 200 + nu)
    rows = _run_modes(cfg, net, p64, x, h, n_list, kernel, 2000 + nu)
    _dump("decode_forms_%s_nu%d.json" % (kernel, nu), {"B": B, "modes": rows, "tol": TOL_64})
    print("%s NU=%d B=%d: max logit err %s (tol %.1e)" % (kernel, nu, B, {m: "%.2e" % r["max_err"] for m, r in
                                                                          rows.items()}, TOL_64))
    for m, r in rows.items():
        assert not r["bad_picks"], (m, r["bad_picks"])
        assert r["max_err"] <= TOL_64, (m, r["max_err"])


RECIPES = {"ljspeech_ks3": (256, 80, 512, 256, 10, 1, 3, 256), "arctic_512": (256, 28, 512, 256, 10, 3, 2, 80)}


@pytest.mark.parametrize("kernel", ["stream", "direct"])
@pytest.mark.parametrize("recipe", list(RECIPES))
def test_stream_direct_recipe_sizes_vs_fp64(kernel, recipe):
    """512 res / 256 skip at full dilation range (d up to 512: the kernel-size-3 queues hold 2 x 512 slots and wrap),
    >= 64 free-running steps after the warm-up over the receptive field"""
    cfg, net, p64 = _model(RECIPES[recipe])
    rng = np.random.RandomState(5)
    B, T0 = 3, 3
    U = cfg.upsampling_factor
    x = rng.randint(0, 256, size=(B, T0)).astype(np.int64)
    h = rng.standard_normal((B, cfg.n_aux, (T0 + 72 + U - 1) // U + 1)).astype(np.float32)
    n_list = [72, 64, 33]
    rows = _run_modes(cfg, net, p64, x, h, n_list, kernel, 3000)
    _dump("decode_forms_%s_%s.json" % (kernel, recipe), {"cfg": RECIPES[recipe], "modes": rows, "tol": TOL_512})
    print("%s %s: max logit err %s (tol %.1e)" % (kernel, recipe, {m: "%.2e" % r["max_err"] for m, r in rows.items()},
                                                  TOL_512))
    for m, r in rows.items():
        assert not r["bad_picks"], (m, r["bad_picks"])
        assert r["max_err"] <= TOL_512, (m, r["max_err"])


# ---------------------------------------------------------------------------------------------------------------------
# long runs: 10 000 sampled steps with in-kernel Philox at the bench shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["warp_cl2", "warp_cl1", "stream", "direct"])
def test_long_sampling_run_vs_fp64(which):
    """The decoder state is a function of the sample history only, so its fp32 error must not grow along the run: the
    worst error of the last 1 000 steps may exceed that of the first 1 000 by no more than the bound."""
    cfg, net, p64 = _model(BENCH)
    n = 10000
    nsm = _nsm()
    B = nsm // 2 + 1 if which == "warp_cl1" else 3
    rng = np.random.RandomState(21)
    x = rng.randint(0, 256, size=(B, 2)).astype(np.int64)
    h = rng.standard_normal((B, 28, (n + 2 + 79) // 80 + 1)).astype(np.float32)
    n_list = [n, n - 1000, n] + [int(v) for v in rng.randint(1, 50, size=B - 3)]
    kernel = "warp" if which.startswith("warp") else which
    if kernel == "warp":
        assert _warp_form(B, 30) == ((1, 16, 2, 1) if which == "warp_cl2" else (1, 16, 1, 1))
    seed = 777
    gen, lg = _decode(net, x, h, n_list, "sampling", kernel, seed=seed)
    uni = D.philox_uniform(seed, np.arange(B)[:, None], np.arange(n)[None, :])
    err, bad = _check(cfg, p64, x, h, n_list, gen, lg, "sampling", uni)
    first, last = np.nanmax(err[:3, :1000]), np.nanmax(np.stack([err[b, n_list[b] - 1000:n_list[b]] for b in range(3)]))
    rep = {"B": B, "n": n, "max_err": float(np.nanmax(err)), "first_1000": float(first), "last_1000": float(last),
           "bad_picks": bad, "tol": TOL_64}
    _dump("decode_forms_long_%s.json" % which, rep)
    print("long sampling run %s (B=%d, %d steps): max logit err %.2e, first 1000 %.2e, last 1000 %.2e (tol %.1e)"
          % (which, B, n, rep["max_err"], first, last, TOL_64))
    assert not bad, bad
    assert rep["max_err"] <= TOL_64
    assert last <= first + TOL_64


# ---------------------------------------------------------------------------------------------------------------------
# CDF-boundary sweep
# ---------------------------------------------------------------------------------------------------------------------
# the bf16 decoder's own pick (decode_bf16.cu): arctic at B = 64, where every CTA's 4 warps pick 2 rows each, and
# 256/256 at B = 70, two clusters of 35
BF16_SWEEP = {"arctic_B64": ((256, 28, 512, 256, 10, 3, 2, 80), 64), "r256_B70": ((256, 28, 256, 256, 4, 2, 2, 4), 70)}
SWEEP = [("warp", f) for f in WARP_FORMS if f not in ("speaker_A31_U0", "A32", "split8")] + \
        [(k, "nu%d" % nu) for k in ("stream", "direct") for nu in (1, 2, 4)] + [("bf16", f) for f in BF16_SWEEP]


@pytest.mark.parametrize("kernel,form_id", SWEEP)
def test_sampling_cdf_boundary_sweep(kernel, form_id, monkeypatch):
    """Step 0's logits do not depend on the uniforms: one launch gets them, then the same inputs are decoded once per
    uniform, with uni * total within +-8 ulps of each of the 31 lane boundaries (and uni = 0, 1 - 2^-24), a different
    uniform for every utterance of a batch.  Every pick must be admissible, so of nonzero probability."""
    if kernel == "warp":
        cfg, net, p64, B, form = _setup_warp(form_id, monkeypatch)
    elif kernel == "bf16":
        t, B = BF16_SWEEP[form_id]
        cfg, net, p64 = _model(t)
        form = form_id
    else:
        cfg, net, p64 = _model(SHALLOW)
        nsm = _nsm()
        B = {"nu1": 64, "nu2": nsm + 5, "nu4": 2 * nsm + 5}[form_id]
        form = form_id
    x, h, _ = _inputs(cfg, B, 3, 1, 300 + len(form_id))
    n_list = [1] * B
    _, lg0 = _decode(net, x, h, n_list, "argmax", kernel)
    ulist = [D.boundary_uniforms(lg0[b, 0]) for b in range(B)]
    K = max(u.size for u in ulist)
    bad, n_draws = [], 0
    for j in range((K + B - 1) // B):
        uni = np.array([[u[(j * B + b) % u.size]] for b, u in enumerate(ulist)], np.float32)
        gen, lg = _decode(net, x, h, n_list, "sampling", kernel, uniforms=uni)
        assert np.array_equal(lg[:, 0], lg0[:, 0])          # step 0 is independent of the uniforms
        ok = D.admissible(lg[:, 0], uni[:, 0])[np.arange(B), gen[:, 0]]
        n_draws += B
        for b in np.nonzero(~ok)[0]:
            bad.append({"utt": int(b), "uni": float(uni[b, 0]), "pick": int(gen[b, 0]),
                        "p_pick": float(np.exp(np.float64(lg[b, 0, gen[b, 0]]) - lg[b, 0].max())
                                        / np.exp(lg[b, 0].astype(np.float64) - lg[b, 0].max()).sum())})
    picks255 = sum(1 for r in bad if r["pick"] == 255)
    _dump("decode_forms_sweep_%s_%s.json" % (kernel, form_id), {"B": B, "form": form, "draws": n_draws,
                                                                 "bad": bad[:50], "n_bad": len(bad)})
    print("CDF-boundary sweep %s %s (form %s, B=%d): %d draws, %d inadmissible (%d of them class 255)"
          % (kernel, form_id, form, B, n_draws, len(bad), picks255))
    assert not bad, (len(bad), picks255, bad[:10])
