#!/usr/bin/env python
"""Per-kernel GPU time of one training step of the bench workload (bench.py's model and batch), from torch.profiler.

    python tools/kernel_times.py [--steps N] [--match SUBSTRING ...]

Prints one line per kernel name: total microseconds per step and launches per step, sorted by time; with --match only
the kernels whose name contains one of the substrings (e.g. the fixed-order reductions: --match front_embed token_kernel
sum_rows sum_loss wgrad_reduce aux_upsample_bwd).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--match", nargs="*", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.optim import Adam
    dev = torch.device("cuda", 0)
    cfg, net = bench.make_model(dev, "tf32")
    net.train()
    opt = Adam(net.parameters(), lr=1e-4, module=net)
    x, h, t = (a.to(dev) for a in bench.synth_batch(cfg, 0, bench.BATCH, pinned=False))

    def step():
        loss = net.forward_loss(x, h, t, cfg.receptive_field)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        if getattr(e, "self_device_time_total", 0) <= 0 or e.count == 0:   # GPU kernels only
            continue
        if args.match and not any(m in e.key for m in args.match):
            continue
        rows.append((e.self_device_time_total / args.steps, e.count / args.steps, e.key))
    for us, n, name in sorted(rows, reverse=True):
        print("%10.1f us/step %6.1f launches/step  %s" % (us, n, name[:110]))
    print("%10.1f us/step in the kernels listed" % sum(r[0] for r in rows))


if __name__ == "__main__":
    main()
