#!/usr/bin/env python
"""Per-kernel GPU time of one training step of the bench workload (bench.py's model and batch), from torch.profiler.

    python tools/kernel_times.py [--steps N] [--match SUBSTRING ...] [--math {tf32,bf16,fp32}]
                                 [--cfg Q,A,R,S,depth,repeat,ks,U --batch B --length T]

Prints one line per kernel name: total microseconds per step and launches per step, sorted by time; with --match only
the kernels whose name contains one of the substrings (e.g. the fixed-order reductions: --match front_embed token_kernel
sum_rows sum_loss wgrad_reduce aux_upsample_bwd).  --math picks the model's math_mode, --cfg another architecture (e.g.
the recipe shapes 256,28,512,256,10,3,2,80 --length 23040 or 256,80,512,256,10,3,3,256 --length 20992) on random
weights and a random batch of --batch windows.
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
    ap.add_argument("--math", default="tf32", choices=["tf32", "bf16", "fp32"])
    ap.add_argument("--cfg", default=None, help="Q,A,R,S,depth,repeat,ks,U (default: bench.py's model and batch)")
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    ap.add_argument("--length", type=int, default=None, help="samples per window with --cfg (a multiple of U)")
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.optim import Adam
    dev = torch.device("cuda", 0)
    if args.cfg is None:
        cfg, net = bench.make_model(dev, args.math)
        x, h, t = (a.to(dev) for a in bench.synth_batch(cfg, 0, args.batch, pinned=False))
    else:
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from math_mode_times import make
        c = tuple(int(v) for v in args.cfg.split(","))
        if args.length is None:
            raise SystemExit("--length is required with --cfg")
        net, _ = make(c, args.math, dev)
        cfg = bench._Cfg(c)
        g = torch.Generator().manual_seed(20260924)
        xfull = torch.randint(0, c[0], (args.batch, args.length + 1), generator=g, dtype=torch.int64)
        x, t = xfull[:, :-1].contiguous().to(dev), xfull[:, 1:].contiguous().to(dev)
        h = torch.randn(args.batch, c[1], args.length // max(c[7], 1), generator=g).to(dev)
    net.train()
    opt = Adam(net.parameters(), lr=1e-4, module=net)

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
