#!/usr/bin/env python
"""Time the stack's weight-gradient phase (dW1, dW2res, dWskip and their biases: one launch + reduce, profile kind
WNB_PROF_WGRAD) at bench.py's training shape, with its algorithmic HBM bytes, HBM rate and tf32 TFLOP/s.

    python tools/wgrad_times.py [--steps N] [--batch B]

Bytes are bench.py's per-kind algorithmic bytes summed (dpre_l, x_l, aux | dout_l, z_l | dskip, Z_all, each streamed
once); FLOPs are 2 B T (L 2R K1 + (L-1) R R + S L R).  A library without the merged kind (the three separate
launches of older builds) is timed as the sum of its dw1, dw2res and dwskip kinds.  Prints the card, its power limit
and SM clock in the same call.
"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tools.gemm_traffic import card  # noqa: E402

PROF_WGRAD = 8                       # WNB_PROF_WGRAD (include/wnb200.h)
PROF_PARTS = (5, 6, 7)               # WNB_PROF_DW1, _DW2RES, _DWSKIP


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    args = ap.parse_args()
    import torch
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.optim import Adam
    print("card, power limit, SM clock, max SM clock:", card())
    dev = torch.device("cuda", 0)
    cfg, net = bench.make_model(dev, "tf32")
    x, h, t = (a.to(dev) for a in bench.synth_batch(cfg, 0, args.batch, pinned=False))
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
    lib = _lib.load()
    _lib.check(lib.wnb_profile_enable(1), "profile_enable")
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()

    def read(kind):
        tot, n = ctypes.c_double(0.0), ctypes.c_int(0)
        if lib.wnb_profile_read(kind, ctypes.byref(tot), ctypes.byref(n)) != 0:
            return None
        return tot.value, n.value

    merged = read(PROF_WGRAD)
    if merged is not None and merged[1] > 0:
        ms, form = merged[0] / args.steps, "one launch (WNB_PROF_WGRAD)"
    else:
        ms, form = sum(read(k)[0] for k in PROF_PARTS) / args.steps, "sum of the dw1, dw2res, dwskip launches"
    _lib.check(lib.wnb_profile_enable(0), "profile_enable")
    Q, A, R, S, depth, repeat, ks, _ = bench.CFG
    Ap, L = (A + 31) // 32 * 32, depth * repeat
    K1 = ks * R + Ap
    Bq, T = x.shape
    bt4 = float(Bq) * T * 4
    hbm = (L * bt4 * 3 * R + bt4 * Ap) + (L - 1) * bt4 * 2 * R + bt4 * (S + L * R)
    flops = 2.0 * Bq * T * (L * 2 * R * K1 + (L - 1) * R * R + S * L * R)
    print("shape: batch %d x %d samples, %d blocks" % (Bq, T, L))
    print("weight gradients (%s): %.3f ms per step, %.2f GB -> %.0f GB/s, %.1f GFLOP -> %.1f TFLOP/s"
          % (form, ms, hbm / 1e9, hbm / (ms * 1e-3) / 1e9, flops / 1e9, flops / (ms * 1e-3) / 1e12))


if __name__ == "__main__":
    main()
