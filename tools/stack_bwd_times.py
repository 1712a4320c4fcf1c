#!/usr/bin/env python
"""Time the block chain of the stack backward (profile kind WNB_PROF_GATE_BWD: the last block's gate backward, one
stack_bwd_chain launch per block boundary -- dx_l and the gate backward of block l-1 -- and dx_0) at bench.py's
training shape, with its algorithmic HBM bytes and HBM rate.

    python tools/stack_bwd_times.py [--steps N] [--batch B]

Algorithmic bytes (fp32 channels-last tensors, each streamed once; weights not counted), per launch:
  boundary launch   (8R + 3Ap) 4 B T: dpre_l 2R, dx_{l+1} R, dx_l out R, dhaux read + write 2Ap, x_{l-1} R, aux Ap,
                    dZ_all slice R, dpre_{l-1} out 2R (the first boundary has no dx_{l+1}: R less)
  last gate alone   (4R + Ap) 4 B T;   dx_0 alone   (4R + 2Ap) 4 B T
A library that still runs the two launches per block (WNB_PROF_DX_GEMM has launches) is timed as the sum of the two
kinds, with bench.py's bytes for them (gate backward (5R + Ap), dX (4R + 2Ap), the last block's gate backward R less).
Prints the card, its power limit and SM clock in the same call.
"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tools.gemm_traffic import card  # noqa: E402

PROF_GATE_BWD = 3                    # WNB_PROF_GATE_BWD (include/wnb200.h)
PROF_DX_GEMM = 4                     # WNB_PROF_DX_GEMM: launched only by libraries without the chain kernel


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
        _lib.check(lib.wnb_profile_read(kind, ctypes.byref(tot), ctypes.byref(n)), "profile_read")
        return tot.value / args.steps, n.value // args.steps

    gate_ms, gate_n = read(PROF_GATE_BWD)
    dx_ms, dx_n = read(PROF_DX_GEMM)
    _lib.check(lib.wnb_profile_enable(0), "profile_enable")
    Q, A, R, S, depth, repeat, ks, _ = bench.CFG
    Ap, L = (A + 31) // 32 * 32, depth * repeat
    Bq, T = x.shape
    bt4 = float(Bq) * T * 4
    print("shape: batch %d x %d samples, %d blocks" % (Bq, T, L))
    if dx_n == 0:
        per_launch = bt4 * (8 * R + 3 * Ap)
        hbm = bt4 * (4 * R + Ap) + (L - 1) * per_launch - (bt4 * R if L > 1 else 0) + bt4 * (4 * R + 2 * Ap)
        print("block chain, %d launches per step (last gate backward, %d boundary launches, dx_0): %.3f ms per step, "
              "%.2f GB -> %.0f GB/s" % (gate_n, L - 1, gate_ms, hbm / 1e9, hbm / (gate_ms * 1e-3) / 1e9))
        print("boundary launch: %.1f MB algorithmic, mean chain launch %.3f ms" % (per_launch / 1e6, gate_ms / gate_n))
    else:
        hbm_g, hbm_x = L * bt4 * (5 * R + Ap) - bt4 * R, L * bt4 * (4 * R + 2 * Ap)
        ms = gate_ms + dx_ms
        print("gate backward: %d launches, %.3f ms per step, %.0f GB/s; dX: %d launches, %.3f ms per step, %.0f GB/s"
              % (gate_n, gate_ms, hbm_g / (gate_ms * 1e-3) / 1e9, dx_n, dx_ms, hbm_x / (dx_ms * 1e-3) / 1e9))
        print("block chain (two launches per block): %.3f ms per step, %.2f GB -> %.0f GB/s"
              % (ms, (hbm_g + hbm_x) / 1e9, (hbm_g + hbm_x) / (ms * 1e-3) / 1e9))


if __name__ == "__main__":
    main()
