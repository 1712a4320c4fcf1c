# -*- coding: utf-8 -*-
"""Held-out scoring (WaveNet.score through utils.scoring.score_utterances), timed.

    python tools/evaluate_times.py [--json out.json]

Random weights and random codes / features; every timed region ends in a synchronise, after an untimed run of the same
shapes.  Reported:
  a. 64 utterances of 10 s (160 000 samples at 16 kHz) at the BASELINE 64/512 shape under tf32, and at the arctic
     512/256 shape under tf32 and bf16, with the --batch_samples default (2^19);
  b. one dev evaluation of an arctic-sized held-out list (64 utterances of 3 s) at arctic tf32, next to one training
     step of the recipe's batch (--batch_length 20 000, --batch_size 1 at rf 3 070) on the same model: zero_grad,
     forward_loss, backward and the Adam step of bin/train.py;
  c. the wnb_cross_entropy_rows launch alone against the no-grad forward of one scoring batch (3 rows of 10 s, the
     2^19-sample budget) at 64/512 and arctic tf32, and of one window row (1 x 524 240 samples), CUDA events, median
     of 5.
Prints the card and its power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BASE = (256, 28, 64, 512, 10, 3, 2, 80)
ARCTIC = (256, 28, 512, 256, 10, 3, 2, 80)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except Exception:   # noqa: BLE001 -- no nvidia-smi: report the name only
        q = "?"
    return "%s (power limit, SM clock: %s)" % (name, q)


def model(shape, mode):
    from pytorchwavenetvocoder_b200.nets import WaveNet, initialize
    torch.manual_seed(0)
    net = WaveNet(*shape)
    net.apply(initialize)
    net.math_mode = mode
    return net.cuda()


def utts(n, T, shape, seed=0):
    rng = np.random.RandomState(seed)
    U = shape[7]
    out = []
    for _ in range(n):
        c = rng.randint(0, 256, size=T + 1).astype(np.int64)
        out.append((c[:T], c[1:], rng.standard_normal((shape[1], T // U)).astype(np.float32)))
    return out


def timed(fn, reps=1):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.utils.scoring import score_utterances
    res = {"card": card()}
    print(res["card"])
    budget = 1 << 19
    ten = utts(64, 160000, BASE)
    for name, shape, mode in (("base_64_512", BASE, "tf32"), ("arctic_512_256", ARCTIC, "tf32"),
                              ("arctic_512_256", ARCTIC, "bf16")):
        net = model(shape, mode)
        s = timed(lambda: score_utterances(net, ten, budget))
        res["a_%s_%s_s" % (name, mode)] = s
        print("a. 64 x 10 s at %s %s: %.3f s (%.1f k samples / s)" % (name, mode, s, 64 * 160000 / s / 1e3))
        del net
        torch.cuda.empty_cache()
    net = model(ARCTIC, "tf32")
    dev = utts(64, 48000, ARCTIC, 1)
    s = timed(lambda: score_utterances(net, dev, budget))
    res["b_arctic_dev_64x3s_tf32_s"] = s
    rf = net.receptive_field
    T = (rf + 20000) // 80 * 80
    rng = np.random.RandomState(2)
    x = torch.from_numpy(rng.randint(0, 256, size=(1, T))).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(1, T))).cuda()
    h = torch.from_numpy(rng.standard_normal((1, 28, T // 80)).astype(np.float32)).cuda()
    net.train()
    from pytorchwavenetvocoder_b200.optim import Adam
    opt = Adam(net.parameters(), lr=1e-4, module=net)

    def step():
        opt.zero_grad()
        net.forward_loss(x, h, t, rf).backward()
        opt.step()
    st = timed(step, 10)
    res["b_arctic_train_step_tf32_s"] = st
    print("b. arctic tf32: one dev evaluation of 64 x 3 s: %.3f s; one training step with Adam (1 x %d): %.1f ms "
          "(%.1f steps)"
          % (s, T, st * 1e3, s / st))
    del net, opt
    torch.cuda.empty_cache()
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    for name, shape in (("base_64_512", BASE), ("arctic_512_256", ARCTIC)):
        net = model(shape, "tf32")
        for B, T in ((3, 160000), (1, (1 << 19) // 80 * 80)):
            rng = np.random.RandomState(3)
            xb = torch.from_numpy(rng.randint(0, 256, size=(B, T))).cuda()
            tb = torch.from_numpy(rng.randint(0, 256, size=(B, T))).cuda()
            hb = torch.from_numpy(rng.standard_normal((B, 28, T // 80)).astype(np.float32)).cuda()
            lengths = torch.full((B,), T, dtype=torch.int64, device="cuda")
            nll = torch.zeros(B, dtype=torch.float64, device="cuda")
            cnt = torch.zeros(B, dtype=torch.int64, device="cuda")
            with torch.no_grad():
                logits = net(xb, hb)

            def ce():
                _lib.check(lib.wnb_cross_entropy_rows(logits.data_ptr(), tb.data_ptr(), lengths.data_ptr(),
                                                      net.receptive_field, nll.data_ptr(), cnt.data_ptr(), B, T, 256,
                                                      _lib.stream()), "cross_entropy_rows")

            def fw():
                with torch.no_grad():
                    net(xb, hb)
            ms = {}
            for what, fn in (("ce", ce), ("forward", fw)):
                fn()
                runs = []
                for _ in range(5):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    runs.append(e0.elapsed_time(e1))
                ms[what] = sorted(runs)[2]
            res["c_%s_%dx%d_ce_ms" % (name, B, T)] = ms["ce"]
            res["c_%s_%dx%d_forward_ms" % (name, B, T)] = ms["forward"]
            print("c. %s tf32, %d x %d: cross_entropy_rows %.3f ms, no-grad forward %.1f ms (%.1f %%)"
                  % (name, B, T, ms["ce"], ms["forward"], 100 * ms["ce"] / ms["forward"]))
            del logits
        del net
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
