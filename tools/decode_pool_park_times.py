# -*- coding: utf-8 -*-
"""Parking and cancelling streams of a bf16 decode pool (WaveNet.decode_pool(park_below=m)): what they cost and what
they buy when clients stall.

    python tools/decode_pool_park_times.py [--requests 96] [--interval-ms 20] [--bound-s 20] [--json out.json]

Shape: arctic 512/256 (256,28,512,256,10,3,2,80: rf 3 070, 80-sample frames, decode_math = "bf16"), Philox sampling,
one-sample seeds, 64 rows.  Reported:
  1. wnb_decode_bf16_pool_park and wnb_decode_bf16_pool_unpark of 1, 8 and 64 streams (3.1 MB each way per stream):
     CUDA events around 20 launches, after one untimed launch; the median of --reps;
  2. the workload of tools/decode_pool_times.py (--requests requests of 800-3 200 samples, one every --interval-ms, the
     pool stepping 100 samples per call), with clients that send their aux as it is made, at 16 k samples/s from arrival.
     Every 8th client stalls for 1 s mid-utterance: it sends the first half of its frames, and the rest 1 s after the
     pool has fewer than 80 of its samples left to run.  Client 5 disconnects after its first half; the parking pools
     cancel it 1 s after they have fewer than 80 of its samples left to run.  Lock step (park_below=None, which has no cancel here: the stream holds its row) against
     park_below=1 and park_below=80.  Reported for the healthy clients (neither stalling nor disconnected): completed
     samples/s and the mean and p95 completion time (arrival to last sample on the device).  A lock-step run never
     finishes once the disconnected client holds back every row, so every run stops after --bound-s seconds and reports
     what it completed.
Prints the card, its power limit and its SM clock, read in the same run."""
import argparse
import ctypes
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
RATE = 16000.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                           timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return name, q or "unavailable"


def model():
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    net = WaveNet(*CFG).cuda().eval()
    net.decode_math = "bf16"
    return net


def park_times(net, reps):
    """{G: (park ms, unpark ms)} per launch of G streams"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import check, ptr, stream
    lib = _lib.load()
    pool = net.decode_pool(64, "sampling", 1)
    nbytes = lib.wnb_decode_bf16_park_bytes(pool.R, pool.ks, pool.dil, pool.L)
    stores = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(64)]
    out = {}
    for G in (1, 8, 64):
        slots = (ctypes.c_int32 * G)(*range(G))
        rot = (ctypes.c_int32 * G)(*[37 * k for k in range(G)])
        st = (ctypes.c_void_p * G)(*[ptr(t) for t in stores[:G]])

        def park():
            check(lib.wnb_decode_bf16_pool_park(ptr(pool.queues), 64, slots, st, rot, G, pool.R, pool.ks, pool.dil,
                                                pool.L, stream()), "park")

        def unpark():
            check(lib.wnb_decode_bf16_pool_unpark(st, ptr(pool.queues), 64, slots, rot, G, pool.R, pool.ks, pool.dil,
                                                  pool.L, stream()), "unpark")
        res = []
        for fn in (park, unpark):
            fn()
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(20):
                    fn()
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1) / 20)
            res.append(sorted(ts)[reps // 2])
        out[G] = tuple(res)
    return out


def workload(net, requests, interval, seed, park_below, bound):
    """One run; returns the healthy clients' numbers and the stalling and disconnected clients' outcome."""
    rng = np.random.RandomState(seed)
    reqs = []
    for r in range(requests):
        n = int(rng.randint(800, 3201))
        reqs.append((r * interval, n, torch.randn(28, n // 80 + 2, device="cuda")))
    stalling = {r for r in range(requests) if r % 8 == 7}
    gone = 5 if requests > 5 else None
    healthy = [r for r in range(requests) if r not in stalling and r != gone]
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    pool = net.decode_pool(64, "sampling", seed, park_below=park_below)
    sent = {}           # r -> frames sent
    half_at = {}        # r -> time the pool ran short of the first half (stalling and disconnected clients)
    done = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    nxt = 0
    while len(done) < requests:
        now = time.perf_counter() - t0
        if now > bound:
            break
        while nxt < requests and reqs[nxt][0] <= now:
            pool.admit(x, reqs[nxt][1], stream=nxt)
            sent[nxt] = 0
            nxt += 1
        for r in list(sent):
            if pool.finished(r):
                continue
            t_arr, n, h = reqs[r]
            nf = h.size(1)
            want = min(nf, int((now - t_arr) * RATE / 80) + 1)   # real time from arrival
            if r in stalling or r == gone:
                st = pool._sched.streams[r]
                if sent[r] == nf // 2 and st.runnable(pool.U, pool.ks) < 80 and r not in half_at:
                    half_at[r] = now
                if r == gone:
                    want = min(want, nf // 2)
                    if park_below is not None and r in half_at and now >= half_at[r] + 1.0:
                        pool.cancel(r)
                        done[r] = None
                        continue
                elif r not in half_at or now < half_at[r] + 1.0:
                    want = min(want, nf // 2)
            if want > sent[r]:
                pool.feed(r, h[:, sent[r]:want])
                sent[r] = want
        out = pool.step(100)
        if not out:
            time.sleep(0.0005)
            continue
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for k in out:
            if pool.finished(k) and k not in done:
                done[k] = now
    torch.cuda.synchronize()
    span = time.perf_counter() - t0
    fin = [r for r in healthy if done.get(r) is not None]
    lat = np.array([done[r] - reqs[r][0] for r in fin]) if fin else np.array([float("nan")])
    last = max(done[r] for r in fin) if len(fin) == len(healthy) else span
    return dict(healthy=len(healthy), healthy_done=len(fin),
                healthy_samples_per_s=sum(reqs[r][1] for r in fin) / last, mean_s=float(lat.mean()),
                p95_s=float(np.percentile(lat, 95)), stalling_done=sum(done.get(r) is not None for r in stalling),
                stalling=len(stalling), cancelled=gone is not None and gone in done and done[gone] is None,
                span_s=span)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--requests", type=int, default=96)
    ap.add_argument("--interval-ms", type=float, default=20.0)
    ap.add_argument("--bound-s", type=float, default=20.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_pool_park_times.py measures on the GPU: no CUDA device found")
    name, q = card()
    print("card: %s, power limit, SM clock, max SM clock: %s" % (name, q))
    net = model()
    res = {"card": name, "power_limit_sm_clock_max_sm_clock": q}
    with torch.no_grad():
        pt = park_times(net, a.reps)
        res["park_unpark_ms"] = {str(g): dict(park=p, unpark=u) for g, (p, u) in pt.items()}
        print("1. per launch: " + ", ".join("%d streams park %.3f ms / unpark %.3f ms" % (g, p, u)
                                            for g, (p, u) in pt.items()))
        workload(net, 16, a.interval_ms / 1e3, 1, 1, 10.0)   # loads every kernel and shape once
        for m in (None, 1, 80):
            w = workload(net, a.requests, a.interval_ms / 1e3, 7, m, a.bound_s)
            what = "lock step" if m is None else "park_below=%d" % m
            res[what] = w
            print("2. %s: healthy %d/%d done, %.0f samples/s, completion mean %.2f s, p95 %.2f s; stalling %d/%d done; "
                  "disconnected client cancelled: %s; run %.1f s"
                  % (what, w["healthy_done"], w["healthy"], w["healthy_samples_per_s"], w["mean_s"], w["p95_s"],
                     w["stalling_done"], w["stalling"], w["cancelled"], w["span_s"]))
    print("card after the runs: %s, power limit, SM clock, max SM clock: %s" % card())
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
