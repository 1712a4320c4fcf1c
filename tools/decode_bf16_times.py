# -*- coding: utf-8 -*-
"""Decode rate of the recipe-sized models: the fp32 path (decode_math="fp32") against the bf16 tensor-core decoder
(decode_math="bf16", csrc/decode_bf16.cu), alternately in one process.

    python tools/decode_bf16_times.py [--steps 500 1500] [--batches 8 32 64 128] [--json out.json]

Each (shape, B, path) is timed with CUDA events around a synchronised argmax decode at two run lengths; the difference
of the two times over the difference of the lengths is the free-running time per step (the teacher-forced warm-up over
the receptive field, the same in both runs, drops out).  Prints the card, its power limit and SM clock, samples/s and
us per step, and for bf16 the weight bytes one CTA streams per step with the rate that implies."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"arctic 512/256 ks2 A28": (256, 28, 512, 256, 10, 3, 2, 80),
          "ljspeech 512/256 ks3 A80": (256, 80, 512, 256, 10, 1, 3, 256)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit / SM clock unavailable"
    return name, q


def time_decode(net, x, h, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    net._decode(x, h, [n] * x.size(0), "argmax")
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, nargs=2, default=[500, 1500])
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32, 64, 128])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import WaveNet
    lib = _lib.load()
    torch.manual_seed(0)
    name, q = card()
    print("card: %s, power limit / SM clock: %s" % (name, q))
    n1, n2 = args.steps
    rows = []
    for sname, cfg in SHAPES.items():
        Q, A, R, S, depth, repeat, ks, U = cfg
        net = WaveNet(*cfg).cuda().eval()
        L, Ap = depth * repeat, (A + 31) // 32 * 32
        cta_bytes = lib.wnb_decode_bf16_weights(Q, Ap, R, S, ks, L) * 2 // 8
        for B in args.batches:
            rng = np.random.RandomState(B)
            x = torch.from_numpy(rng.randint(0, Q, size=(B, 2))).cuda()
            h = torch.from_numpy(rng.standard_normal((B, A, (n2 + 2) // max(U, 1) + 2)).astype(np.float32)).cuda()
            res = {}
            with torch.no_grad():
                for dm in ("fp32", "bf16"):       # warm both (packing, module load), then alternate
                    net.decode_math = dm
                    time_decode(net, x, h, 8)
                t = {("fp32", n1): 0.0, ("fp32", n2): 0.0, ("bf16", n1): 0.0, ("bf16", n2): 0.0}
                for n in (n1, n2):
                    for dm in ("fp32", "bf16"):
                        net.decode_math = dm
                        t[(dm, n)] = time_decode(net, x, h, n)
                        res[dm + "_kernel"] = net.last_decode_kernel
            for dm in ("fp32", "bf16"):
                us = (t[(dm, n2)] - t[(dm, n1)]) / (n2 - n1) * 1e6
                row = {"shape": sname, "B": B, "path": dm, "kernel": res[dm + "_kernel"], "us_per_step": us,
                       "samples_per_s": B / us * 1e6}
                if dm == "bf16":
                    row["weight_bytes_per_cta_step"] = cta_bytes
                    row["implied_GBps_per_cta"] = cta_bytes / us * 1e-3
                rows.append(row)
                print("%-26s B=%4d %-5s (%-6s) %9.1f us/step %12.0f samples/s%s" % (
                    sname, B, dm, row["kernel"], us, row["samples_per_s"],
                    "   %.1f MB/CTA/step -> %.0f GB/s per CTA" % (cta_bytes / 1e6, row["implied_GBps_per_cta"])
                    if dm == "bf16" else ""))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit_sm_clock": q, "steps": [n1, n2], "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
