# -*- coding: utf-8 -*-
"""Latency of resumable decode sessions (WaveNet.decode_session): per-chunk latency, time to first audio, and the
throughput of chunked against one-shot decoding.

    python tools/decode_session_times.py [--samples 8000] [--batches 1 8 64] [--chunks 1 5 20 100] [--json out.json]

Shapes: the BASELINE 64/512 model (fp32 warp-tiled decoder) and the arctic 512/256 model with decode_math="bf16", both
with 80-sample frames.  For every (shape, B, chunk of F frames) the session is fed F frames per call; each call is timed
on the host around a synchronise (what a streaming caller waits for).  Reported:
  * first audio: session creation and the first call, which also runs the rf - 1 warm-up steps;
  * per-chunk latency: the median of the later calls, and its value per generated sample;
  * throughput: samples / s over the whole session (its creation included), and its ratio to one one-shot call of the
    same length (its weight packing included).
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

SHAPES = {"baseline 64/512 fp32": ((256, 28, 64, 512, 10, 3, 2, 80), "fp32"),
          "arctic 512/256 bf16": ((256, 28, 512, 256, 10, 3, 2, 80), "bf16")}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = "unavailable"
    return name, q or "unavailable"


def oneshot(net, x, h, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    net._decode(x, h, [n] * x.size(0), "sampling", seed=1)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def session(net, x, h, n, F):
    """host time of every step (around a synchronise) and the samples it produced; the first includes creating the
    session (weight packing, queues), which the one-shot path also pays inside its timed call"""
    torch.cuda.synchronize()
    times, counts, f = [], [], 0
    t0 = time.perf_counter()
    s = net.decode_session(x, [n] * x.size(0), "sampling", seed=1)
    while not s.done:
        s.step(h[:, :, f:f + F])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        times.append(t1 - t0)
        t0 = t1
        counts.append(max(s.last_counts))
        f += F
    return times, counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=8000)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--chunks", type=int, nargs="+", default=[1, 5, 20, 100])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    name, q = card()
    print("card: %s, power limit: %s" % (name, q))
    n = args.samples
    rows = []
    with torch.no_grad():
        for sname, (cfg, dm) in SHAPES.items():
            net = WaveNet(*cfg).cuda().eval()
            net.decode_math = dm
            U = cfg[-1]
            for B in args.batches:
                rng = np.random.RandomState(B)
                x = torch.from_numpy(rng.randint(0, 256, size=(B, 1))).cuda()
                h = torch.from_numpy(rng.standard_normal((B, cfg[1], n // U + 2)).astype(np.float32)).cuda()
                oneshot(net, x, h, 64)                      # warm: module load, packing
                session(net, x, h, 2 * U, 1)
                for F in args.chunks:
                    t_one = oneshot(net, x, h, n)             # next to each session: the clock drifts under a power cap
                    times, counts = session(net, x, h, n, F)
                    later = times[1:-1] or times[1:] or times
                    row = {"shape": sname, "B": B, "chunk_frames": F, "chunk_samples": F * U, "calls": len(times),
                           "first_audio_s": times[0], "first_samples": counts[0],
                           "chunk_latency_ms_median": float(np.median(later)) * 1e3,
                           "chunk_latency_us_per_sample": float(np.median(later)) / (F * U) * 1e6,
                           "samples_per_s": B * n / sum(times), "oneshot_samples_per_s": B * n / t_one,
                           "throughput_ratio": t_one / sum(times)}
                    rows.append(row)
                    print("%-22s B=%3d chunk %3d frames (%5d samples): first audio %7.3f s (%d samples), chunk %8.2f ms "
                          "(%6.1f us/sample), %9.0f samples/s = %.3f x one-shot" % (
                              sname, B, F, F * U, row["first_audio_s"], row["first_samples"],
                              row["chunk_latency_ms_median"], row["chunk_latency_us_per_sample"], row["samples_per_s"],
                              row["throughput_ratio"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": q, "samples": n, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
