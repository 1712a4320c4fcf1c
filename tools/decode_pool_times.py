# -*- coding: utf-8 -*-
"""Continuous batching on the bf16 decoder (WaveNet.decode_pool) against what it replaces.

    python tools/decode_pool_times.py [--steps 480] [--requests 96] [--interval-ms 20] [--json out.json]

Shape: arctic 512/256 (256,28,512,256,10,3,2,80: rf 3 070, 80-sample frames, decode_math = "bf16"), Philox sampling,
one-sample seeds.  Every timed call sits between two synchronises, after an untimed call of the same shape.  Reported:
  1. a full pool's step (64 rows, --steps steps, a multiple of the 80-sample frame) against DecodeSession.step of the same steps at B = 64 (the same
     decoder kernel), and the pool's input kernel (wnb_decode_bf16_pool_inputs) on its own;
  2. admission (prefill + transplant) of groups of 1, 8 and 64 streams;
  3. a seeded staggered-arrival workload: --requests requests of 800-3 200 samples (0.05-0.2 s at 16 kHz) with all
     their aux, arriving every --interval-ms; a pool of 64 rows stepping 100 samples per call, against one decode session
     per request on its own CUDA stream with at most 16 in flight.  Completed samples/s and the mean and p95 of the
     completion time (arrival to last sample on the device).
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

CFG = (256, 28, 512, 256, 10, 3, 2, 80)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = "unavailable"
    return name, q or "unavailable"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def model():
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    net = WaveNet(*CFG).cuda().eval()
    net.decode_math = "bf16"
    return net


def step_times(net, n, reps):
    """(pool step, session step, input kernel) seconds for n steps at 64 rows"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import check, ptr, stream
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    nf = (reps + 2) * n // 80 + 2
    h = torch.randn(64, 28, nf, device="cuda")
    pool = net.decode_pool(64, "sampling", 1)
    for k in range(64):
        pool.admit(x, 10 ** 7, h[k])
    pool.step(n)
    pool_t = sorted(timed(lambda: pool.step(n)) for _ in range(reps))[reps // 2]
    s = net.decode_session(torch.zeros(64, 1, dtype=torch.int64, device="cuda"), [10 ** 7] * 64, "sampling", 1)
    s.step(h[:, :, :n // 80])
    f = [n // 80]

    def sess():
        s.step(h[:, :, f[0]:f[0] + n // 80])
        f[0] += n // 80
    sess_t = sorted(timed(sess) for _ in range(reps))[reps // 2]
    lib = _lib.load()
    frames = torch.randn(64, 28, n // 80 + 1, device="cuda")
    table = torch.tensor([[0] * 64, [0] * 64, [0] * 64, list(range(64)), [n] * 64], dtype=torch.int32, device="cuda")
    aux = torch.empty(64, 28, n, device="cuda")
    uni = torch.empty(64, n, device="cuda")

    def inputs():
        for _ in range(100):
            check(lib.wnb_decode_bf16_pool_inputs(ptr(frames), ptr(pool.upw), ptr(pool.upb), ptr(table), ptr(aux),
                                                  ptr(uni), 64, 28, frames.size(2), n, 80, pool.seed, stream()), "inputs")
    inputs()
    inp_t = sorted(timed(inputs) / 100 for _ in range(reps))[reps // 2]
    return pool_t, sess_t, inp_t


def admission_times(net, reps):
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import PoolStream
    lib = _lib.load()
    pool = net.decode_pool(64, "sampling", 1)
    h = torch.randn(28, 4, device="cuda")
    out = {}
    for G in (1, 8, 64):
        def admit():
            group = []
            for k in range(G):
                st = PoolStream(k, 1, 100, net.receptive_field)
                st.slot = k
                pool._x[k] = torch.zeros(1, dtype=torch.int32, device="cuda")
                pool._h[k] = [h, 0]
                group.append(st)
            pool._admit_group(lib, 1, group, 5)
        admit()
        out[G] = sorted(timed(admit) for _ in range(reps))[reps // 2]
    return out


def workload(net, requests, interval, seed, use_pool):
    rng = np.random.RandomState(seed)
    reqs = []
    for r in range(requests):
        n = int(rng.randint(800, 3201))
        reqs.append((r * interval, n, torch.randn(28, n // 80 + 2, device="cuda")))
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    done = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if use_pool:
        pool = net.decode_pool(64, "sampling", seed)
        nxt = 0
        while len(done) < requests:
            now = time.perf_counter() - t0
            while nxt < requests and reqs[nxt][0] <= now:
                pool.admit(x, reqs[nxt][1], reqs[nxt][2], stream=nxt)
                nxt += 1
            out = pool.step(100)
            if not out:
                time.sleep(0.0005)
                continue
            torch.cuda.synchronize()
            now = time.perf_counter() - t0
            for k in out:
                if pool.finished(k) and k not in done:
                    done[k] = now
    else:
        streams = [torch.cuda.Stream() for _ in range(16)]
        free, flight, nxt = list(range(16)), {}, 0
        while len(done) < requests:
            now = time.perf_counter() - t0
            while nxt < requests and reqs[nxt][0] <= now and free:
                slot = free.pop()
                with torch.cuda.stream(streams[slot]), torch.no_grad():
                    s = net.decode_session(x[None], [reqs[nxt][1]], "sampling", seed + nxt)
                    s.step(reqs[nxt][2][None])
                    ev = torch.cuda.Event()
                    ev.record()
                flight[nxt] = (slot, ev, s)
                nxt += 1
            for r, (slot, ev, s) in list(flight.items()):
                if ev.query():
                    done[r] = time.perf_counter() - t0
                    free.append(slot)
                    del flight[r]
            time.sleep(0.0005)
    lat = np.array([done[r] - reqs[r][0] for r in range(requests)])
    total = sum(n for _, n, _ in reqs)
    return dict(samples_per_s=total / max(done.values()), mean_s=float(lat.mean()), p95_s=float(np.percentile(lat, 95)),
                span_s=max(done.values()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=480)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--requests", type=int, default=96)
    ap.add_argument("--interval-ms", type=float, default=20.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit: %s" % (name, power))
    net = model()
    res = {"card": name, "power_limit": power}
    with torch.no_grad():
        pt, st, it = step_times(net, a.steps, a.reps)
        res["step"] = dict(steps=a.steps, pool_ms=pt * 1e3, session_ms=st * 1e3, inputs_kernel_ms=it * 1e3)
        print("1. %d steps at 64 rows: pool %.1f ms (%.0f us/step), session %.1f ms (%.0f us/step); input kernel %.3f ms"
              % (a.steps, pt * 1e3, pt / a.steps * 1e6, st * 1e3, st / a.steps * 1e6, it * 1e3))
        adm = admission_times(net, a.reps)
        res["admission_ms"] = {str(g): v * 1e3 for g, v in adm.items()}
        print("2. admission (prefill + transplant): " + ", ".join("%d: %.1f ms" % (g, v * 1e3) for g, v in adm.items()))
        workload(net, 8, a.interval_ms / 1e3, 1, True)    # loads every kernel and shape once
        workload(net, 8, a.interval_ms / 1e3, 1, False)
        for what, use_pool in (("pool (64 rows)", True), ("sessions (16 streams)", False)):
            w = workload(net, a.requests, a.interval_ms / 1e3, 7, use_pool)
            res[what] = w
            print("3. %s: %.0f samples/s, completion mean %.2f s, p95 %.2f s (last done at %.2f s)"
                  % (what, w["samples_per_s"], w["mean_s"], w["p95_s"], w["span_s"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
