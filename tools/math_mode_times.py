#!/usr/bin/env python
"""Whole training-step time of math_mode="bf16" against "tf32" at the recipe shapes, in one process.

    python tools/math_mode_times.py [--steps 20] [--warmup 3] [--cfg Q,A,R,S,depth,repeat,ks,U --batch B --length T]

One step = forward + cross entropy + backward + Adam (optim.Adam), timed with CUDA events around each step; the two
modes alternate step by step on the same batch, after a warm-up of both.  Defaults: the arctic recipe
256,28,512,256,10,3,2,80 at 8 x 23 040 samples and the ljspeech-melspc architecture 256,80,512,256,10,3,3,256 at
8 x 20 992 (the SURVEY cfg3 window).  Prints the card name, its power limit and SM clock (read in the same call), the
median step time per mode, the achieved FLOP/s of the whole step (SURVEY 8d formula: forward
L [2R^2 (2ks+1) + 4RA + 2SR] + 2S^2 + 2QS per sample, backward twice that) against the bf16 and tf32 data-sheet rates,
and the loss of the first step of each mode on the same batch.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DATASHEET_TFLOPS = {"bf16": 989.0, "tf32": 495.0}   # H100 SXM, dense, 700 W card
DEFAULT_RUNS = [("256,28,512,256,10,3,2,80", 8, 23040), ("256,80,512,256,10,3,3,256", 8, 20992)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=30)
        return out.stdout.decode().strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s); device %s" % (e, torch.cuda.get_device_name(0))


def step_flops(cfg, B, T):
    Q, A, R, S, depth, repeat, ks, U = cfg
    L = depth * repeat
    fwd = L * (2 * R * R * (2 * ks + 1) + 4 * R * A + 2 * S * R) + 2 * S * S + 2 * Q * S
    return 3.0 * fwd * B * T


def make(cfg, math_mode, dev):
    from pytorchwavenetvocoder_b200.nets import WaveNet, initialize
    from pytorchwavenetvocoder_b200.optim import Adam
    torch.manual_seed(20260924)
    net = WaveNet(*cfg)
    net.apply(initialize)
    with torch.no_grad():
        for name, prm in net.named_parameters():
            if name.endswith("bias"):
                prm.add_(0.05 * torch.randn_like(prm))
    net.math_mode = math_mode
    net = net.to(dev).train()
    return net, Adam(net.parameters(), lr=1e-4, module=net)


def run(cfg, B, T, steps, warmup, dev):
    from pytorchwavenetvocoder_b200.nets.wavenet import bf16_supported
    if not bf16_supported(cfg):
        raise SystemExit("math_mode bf16 does not cover %s" % (cfg,))
    Q, A, U = cfg[0], cfg[1], max(cfg[7], 1)
    rf = (cfg[6] - 1) * sum([2 ** i for i in range(cfg[4])] * cfg[5]) + 1
    g = torch.Generator().manual_seed(20260924)
    xfull = torch.randint(0, Q, (B, T + 1), generator=g, dtype=torch.int64)
    x, t = xfull[:, :-1].contiguous().to(dev), xfull[:, 1:].contiguous().to(dev)
    h = torch.randn(B, A, T // U, generator=g).to(dev)
    models = {m: make(cfg, m, dev) for m in ("tf32", "bf16")}

    def step(m):
        net, opt = models[m]
        loss = net.forward_loss(x, h, t, rf)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss

    first = {m: float(step(m).item()) for m in models}      # same weights, same batch: the first losses compare
    for _ in range(warmup):
        for m in models:
            step(m)
    torch.cuda.synchronize()
    times = {m: [] for m in models}
    for _ in range(steps):
        for m in models:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(m)
            e1.record()
            e1.synchronize()
            times[m].append(e0.elapsed_time(e1))
    flops = step_flops(cfg, B, T)
    print("cfg %s, B %d, T %d (%.1f TFLOP per step, loss from t = %d)" % (",".join(map(str, cfg)), B, T, flops / 1e12, rf))
    for m in ("tf32", "bf16"):
        ms = statistics.median(times[m])
        rate = flops / (ms * 1e-3) / 1e12
        print("  %-4s step %8.2f ms median (min %.2f, max %.2f, %d steps)  %7.1f TFLOP/s whole step = %4.1f %% of the "
              "bf16 / %4.1f %% of the tf32 data-sheet rate" % (m, ms, min(times[m]), max(times[m]), steps, rate,
                                                                100 * rate / DATASHEET_TFLOPS["bf16"],
                                                                100 * rate / DATASHEET_TFLOPS["tf32"]))
    tb, tt = statistics.median(times["bf16"]), statistics.median(times["tf32"])
    print("  bf16 / tf32 step time %.3f; first-step loss bf16 %.6f, tf32 %.6f (difference %.2e)"
          % (tb / tt, first["bf16"], first["tf32"], abs(first["bf16"] - first["tf32"])))
    del models
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cfg", type=str, default=None, help="Q,A,R,S,depth,repeat,ks,U (default: the two recipe shapes)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--length", type=int, default=None, help="samples per window (a multiple of U)")
    args = ap.parse_args()
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    if not torch.cuda.is_available():
        raise SystemExit("math_mode_times needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    print("card: %s" % card())
    runs = DEFAULT_RUNS if args.cfg is None else [(args.cfg, args.batch, args.length)]
    for c, B, T in runs:
        cfg = tuple(int(v) for v in c.split(","))
        if T is None:
            raise SystemExit("--length is required with --cfg")
        run(cfg, B, T, args.steps, args.warmup, dev)
    print("card (after): %s" % card())


if __name__ == "__main__":
    main()
