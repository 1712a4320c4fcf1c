# -*- coding: utf-8 -*-
"""Continuous batching on the fp32 warp decoder (WaveNet.decode_pool with decode_math = "fp32") against what it replaces.

    python tools/decode_pool_fp32_times.py [--steps 480] [--reps 3] [--corpus 256] [--corpus-reps 2] [--parts abcde]
        [--json out.json]

Shape: the BASELINE model, 64 res / 512 skip (256,28,64,512,10,3,2,80: 30 layers, rf 3 070, 80-sample frames), Philox
sampling, one-sample seeds.  Every timed call sits between two synchronises, after an untimed call of the same shape.
Reported:
  a. a full 64-row pool's step (--steps steps) against DecodeSession.step of the same steps at B = 64 (the same warp
     kernel and form: one utterance per 2-CTA cluster), and the pool's input kernel on its own; then, per step at 480
     and 4 800 steps per call, the pool, that session (aux frames, U = 80), a session of the same weights on a U = 0
     model fed sample-rate aux (what the pool feeds the kernel), and the host time of a pool call until it returns
     (nothing synchronises inside a call): a gap that shrinks with the steps per call is per call, one that stays is
     per step;
  b. admission (prefill at the pool's CL + one wnb_decode_pool_move) of groups of 1, 8 and 64 streams;
  c. the park and the unpark launch (wnb_decode_pool_move between pool rows and stores) for 1, 8 and 64 streams;
  d. a corpus of --corpus utterances of 1-6 s at 16 kHz with all their aux: length-sorted batch_fast_generate batches
     of 32 and of 64 against one 64-row pool admitting every utterance longest first; wall time and samples/s, outputs
     not compared, the three runs alternated --corpus-reps times;
  e. the staggered-request workload of tools/decode_pool_times.py (96 requests of 800-3 200 samples every 20 ms): a
     64-row pool against one decode session per request, at most 16 in flight.
Prints the card, its power limit and its SM clock, read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from decode_pool_times import admission_times, step_times, timed, workload   # noqa: E402

CFG = (256, 28, 64, 512, 10, 3, 2, 80)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    parts = [p.strip() for p in q.split(",")] if q else []
    return name, parts[0] if parts else "unavailable", parts[1] if len(parts) > 1 else "unavailable"


def model():
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    net = WaveNet(*CFG).cuda().eval()
    assert net.decode_math == "fp32"
    return net


def step_breakdown(net, reps):
    """{n: dict of us per step (pool, session U 80, session U 0) and host ms per pool call} for n steps per call"""
    from pytorchwavenetvocoder_b200.nets import WaveNet
    net0 = WaveNet(*CFG[:7], 0).cuda().eval()
    net0.load_state_dict({k: v for k, v in net.state_dict().items() if not k.startswith("upsampling")})
    ns = (480, 4800)
    total = (reps + 1) * sum(ns)
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    h = torch.randn(64, 28, total // 80 + 4, device="cuda")
    h0 = torch.randn(64, 28, total + 8, device="cuda")
    pool = net.decode_pool(64, "sampling", 1)
    for k in range(64):
        pool.admit(x, 10 ** 7, h[k])
    s = net.decode_session(torch.zeros(64, 1, dtype=torch.int64, device="cuda"), [10 ** 7] * 64, "sampling", 1)
    s0 = net0.decode_session(torch.zeros(64, 1, dtype=torch.int64, device="cuda"), [10 ** 7] * 64, "sampling", 1)
    f, c = [0], [0]

    def sess(n):
        s.step(h[:, :, f[0]:f[0] + n // 80])
        f[0] += n // 80

    def sess0(n):
        s0.step(h0[:, :, c[0]:c[0] + n])
        c[0] += n
    out = {}
    for n in ns:
        pool.step(n)
        sess(n)
        sess0(n)
        host = []

        def pool_call():
            t = time.perf_counter()
            pool.step(n)
            host.append(time.perf_counter() - t)
        med = lambda fn: sorted(timed(fn) for _ in range(reps))[reps // 2] / n * 1e6
        out[n] = dict(pool_us=med(pool_call), session_us=med(lambda: sess(n)), session_u0_us=med(lambda: sess0(n)),
                      pool_host_ms=sorted(host)[len(host) // 2] * 1e3)
    return out


def move_times(net, reps):
    """{n: (park, unpark) seconds}: one wnb_decode_pool_move of n pool rows into stores, and back"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import ptr
    lib = _lib.load()
    pool = net.decode_pool(64, "sampling", 1)
    out = {}
    for n in (1, 8, 64):
        stores = [torch.empty(pool._park_bytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
        park = [(pool._row(s), ptr(stores[s]), 17 - s) for s in range(n)]
        unpark = [(ptr(stores[s]), pool._row(63 - s), s - 17) for s in range(n)]
        pool._move(lib, park)
        pool._move(lib, unpark)
        out[n] = (sorted(timed(lambda: pool._move(lib, park)) for _ in range(reps))[reps // 2],
                  sorted(timed(lambda: pool._move(lib, unpark)) for _ in range(reps))[reps // 2])
    return out


def corpus(n, seed):
    rng = np.random.RandomState(seed)
    lens = [int(v) for v in rng.randint(16000, 96001, n)]
    return [(m, torch.randn(28, m // 80 + 2, device="cuda")) for m in lens]


def run_batches(net, utts, B):
    order = sorted(range(len(utts)), key=lambda k: utts[k][0])
    t = time.perf_counter()
    for k0 in range(0, len(order), B):
        part = [utts[k] for k in order[k0:k0 + B]]
        nf = max(h.size(1) for _, h in part)
        H = torch.zeros(len(part), 28, nf, device="cuda")
        for b, (_, h) in enumerate(part):
            H[b, :, :h.size(1)] = h
        X = torch.full((len(part), 1), 128, dtype=torch.int64, device="cuda")
        net.batch_fast_generate(X, H, [m for m, _ in part])
    torch.cuda.synchronize()
    return time.perf_counter() - t


def run_pool(net, utts):
    x = torch.full((1,), 128, dtype=torch.int64, device="cuda")
    t = time.perf_counter()
    pool = net.decode_pool(64, "sampling", 3)
    for k in sorted(range(len(utts)), key=lambda k: -utts[k][0]):
        pool.admit(x, utts[k][0], utts[k][1], stream=k)
    while pool.active or pool.waiting:
        pool.step()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=480)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--requests", type=int, default=96)
    ap.add_argument("--interval-ms", type=float, default=20.0)
    ap.add_argument("--corpus", type=int, default=256)
    ap.add_argument("--corpus-reps", type=int, default=2)
    ap.add_argument("--parts", default="abcde", help="which of the reports a-e to run")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    name, power, clock = card()
    print("card: %s, power limit: %s, SM clock: %s" % (name, power, clock))
    net = model()
    res = {"card": name, "power_limit": power, "sm_clock": clock}
    with torch.no_grad():
        if "a" in a.parts:
            pt, st, it = step_times(net, a.steps, a.reps)
            res["a_step"] = dict(steps=a.steps, pool_ms=pt * 1e3, session_ms=st * 1e3, inputs_kernel_ms=it * 1e3)
            print("a. %d steps at 64 rows: pool %.2f ms (%.1f us/step), session %.2f ms (%.1f us/step); input kernel "
                  "%.3f ms" % (a.steps, pt * 1e3, pt / a.steps * 1e6, st * 1e3, st / a.steps * 1e6, it * 1e3))
            bd = step_breakdown(net, a.reps)
            res["a_breakdown"] = {str(n): v for n, v in bd.items()}
            for n, v in bd.items():
                print("a. %d steps per call, us/step: pool %.1f, session (U 80) %.1f, session (U 0, sample-rate aux) "
                      "%.1f; host time of a pool call %.2f ms"
                      % (n, v["pool_us"], v["session_us"], v["session_u0_us"], v["pool_host_ms"]))
        if "b" in a.parts:
            adm = admission_times(net, a.reps)
            res["b_admission_ms"] = {str(g): v * 1e3 for g, v in adm.items()}
            print("b. admission (prefill + move): " + ", ".join("%d: %.2f ms" % (g, v * 1e3) for g, v in adm.items()))
        if "c" in a.parts:
            mv = move_times(net, a.reps)
            res["c_move_ms"] = {str(n): dict(park=p * 1e3, unpark=u * 1e3) for n, (p, u) in mv.items()}
            print("c. park / unpark launch: " + ", ".join("%d: %.3f / %.3f ms" % (n, p * 1e3, u * 1e3)
                                                         for n, (p, u) in mv.items()))
        if "d" in a.parts:
            utts = corpus(a.corpus, 5)
            total = sum(m for m, _ in utts)
            run_batches(net, utts[:4], 4)   # loads every kernel once
            run_pool(net, utts[:4])
            runs = {"batches of 32": [], "batches of 64": [], "pool of 64": []}
            for _ in range(a.corpus_reps):
                runs["batches of 32"].append(run_batches(net, utts, 32))
                runs["batches of 64"].append(run_batches(net, utts, 64))
                runs["pool of 64"].append(run_pool(net, utts))
            res["d_corpus"] = dict(utterances=a.corpus, samples=total,
                                   runs={k: dict(wall_s=v, samples_per_s=[total / t for t in v])
                                         for k, v in runs.items()})
            for k, v in runs.items():
                print("d. %d utterances, %.1f M samples, %s: wall %s s, %s M samples/s"
                      % (a.corpus, total / 1e6, k, " / ".join("%.2f" % t for t in v),
                         " / ".join("%.3f" % (total / t / 1e6) for t in v)))
        if "e" in a.parts:
            workload(net, 8, a.interval_ms / 1e3, 1, True)    # loads every kernel and shape once
            workload(net, 8, a.interval_ms / 1e3, 1, False)
            for what, use_pool in (("pool (64 rows)", True), ("sessions (16 streams)", False)):
                w = workload(net, a.requests, a.interval_ms / 1e3, 7, use_pool)
                res["e " + what] = w
                print("e. %s: %.0f samples/s, completion mean %.3f s, p95 %.3f s (last done at %.2f s)"
                      % (what, w["samples_per_s"], w["mean_s"], w["p95_s"], w["span_s"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
