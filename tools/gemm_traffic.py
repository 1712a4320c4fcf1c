#!/usr/bin/env python
"""Where the bytes of the gemm_nt_tc launches go: per launch kind of the deferred-skip stack and the post network,
the weight and activation bytes the SMs pull from L2, the algorithmic HBM bytes and the tf32 FLOPs.

    python tools/gemm_traffic.py [--cm 1|2|4] [--batch B] [--length T] [--time [--steps N]]

Shapes are bench.py's model (configs[1]: 30 blocks, R = 64, S = 512, Q = 256, A = 28 padded to 32) at --batch windows
of --length samples (default: bench.py's batch, 8 x 23 040).  A gemm_nt_tc work item is a pair of 64-row time tiles
(flattened over the batch) of one column block, and loads that block's whole [N x K] weight operand once for both
tiles; CTAs in a cluster of CM share each weight box (multicast), so the weight column is divided by CM.  Rows a tensor
map zero-fills (the dx launch's shifted segment reads a 64-row matrix through a 96-row box) are not counted.

--time (needs the GPU) runs --steps training steps with CM forced to --cm (WNB_NT_CLUSTER) and wnb_profile_enable(1),
as bench.py's roofline block does, and adds each stack kind's ms per step and the achieved L2->SM rate (weight +
activation bytes over that time).  The post network GEMMs are not profiled kinds: tools/kernel_times.py times them.  It
also times a torch sum over an L2-resident buffer as a reference L2 read rate (a lower bound on what the L2 can
deliver), and prints the card, its power limit and SM clock in the same call.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

TM = 64   # time rows per gemm_nt_tc tile; a work item is two tiles


def kinds(B, T, cm):
    """[(kind, launches per step, weight bytes, activation bytes, HBM bytes, FLOPs) per step]"""
    Q, A, R, S, depth, repeat, ks, _ = bench.CFG
    Ap, L = (A + 31) // 32 * 32, depth * repeat
    K1, bt, ntt, s = ks * R + Ap, B * T, B * -(-T // TM), 4
    npairs = -(-ntt // 2)
    rows = []

    def gemm(name, n, segs, hbm):
        """segs: [(K, weight rows read from memory per tile pair)]; n: N of all column blocks together"""
        nblk = max(1, n // 256) if n > 256 else 1
        w = sum(npairs * rows_ * k * s for k, rows_ in segs) / cm
        a = sum(ntt * nblk * TM * k * s for k, _ in segs)
        f = 2 * bt * n * sum(k for k, _ in segs)
        return [name, w, a, hbm, f]

    LR = L * R
    rows.append([1] + gemm("skip_gemm", S, [(LR, S)], bt * (LR + S) * s))
    # dZ_all: N = L*R in column blocks of 192 (10 blocks at L*R = 1920): the A tile is loaded once per block
    r = gemm("dzall_gemm", LR, [(S, LR)], bt * (S + LR) * s)
    r[2] = ntt * (LR // 192) * TM * S * s
    rows.append([1] + r)
    # gate backward: N = 3R over [x(t-d) | x(t) | aux | dout] (K1 + R); the last block has no dout (N = 2R, K = K1)
    g = [0.0] * 4
    for last in (True,) + (False,) * (L - 1):
        n, k = (2 * R, K1) if last else (3 * R, K1 + R)
        _, w, a, _, f = gemm("", n, [(k, n)], 0)
        g = [g[0] + w, g[1] + a, g[2] + bt * (5 * R + Ap) * s, g[3] + f]
    rows.append([L, "gate_bwd"] + g)
    # dx + dhaux: N = R + Ap over dpre (2R) twice; the shifted segment's weight matrix has R rows (the rest zero fill)
    _, w, a, _, f = gemm("", R + Ap, [(2 * R, R + Ap), (2 * R, R)], 0)
    rows.append([L, "dx_gemm", L * w, L * a, L * bt * (2 * R + R + R + Ap) * s, L * f])
    # post network: relu(skip) -> S -> Q forward, and back (two GEMMs each way)
    post = [("post_fwd_1", S, S), ("post_fwd_2", Q, S), ("post_bwd_dh1", S, Q), ("post_bwd_dskip", S, S)]
    for name, n, k in post:
        rows.append([1] + gemm(name, n, [(k, n)], bt * (n + k) * s))
    return rows


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def time_kinds(B, steps):
    import ctypes
    import torch
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.optim import Adam
    dev = torch.device("cuda", 0)
    cfg, net = bench.make_model(dev, "tf32")
    x, h, t = (a.to(dev) for a in bench.synth_batch(cfg, 0, B, pinned=False))
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
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    ms = {}
    for k, name in enumerate(bench.STACK_KINDS):
        tot, n = ctypes.c_double(0.0), ctypes.c_int(0)
        _lib.check(lib.wnb_profile_read(k, ctypes.byref(tot), ctypes.byref(n)), "profile_read")
        ms[name] = tot.value / steps
    _lib.check(lib.wnb_profile_enable(0), "profile_enable")
    # reference: repeated reads of a 16 MB buffer that stays in the 50 MB L2
    buf = torch.ones(4 << 20, device=dev)
    for _ in range(10):
        buf.sum()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        buf.sum()
    e1.record()
    torch.cuda.synchronize()
    l2 = 200 * buf.numel() * 4 / (e0.elapsed_time(e1) * 1e-3) / 1e9
    return ms, l2, int(x.shape[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cm", type=int, default=1, choices=[1, 2, 4], help="CTAs per cluster sharing a weight box")
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    ap.add_argument("--length", type=int, default=None, help="samples per window (default: bench.py's)")
    ap.add_argument("--time", action="store_true", help="also time the stack kinds on the GPU")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    T = args.length
    if T is None:
        cfg = bench._Cfg(bench.CFG)
        T = (bench.BATCH_LENGTH + cfg.receptive_field) // cfg.upsampling_factor * cfg.upsampling_factor
    ms, l2 = {}, None
    if args.time:
        os.environ["WNB_NT_CLUSTER"] = str(args.cm)   # the timed launches use the CM the bytes are counted for
        print("card, power limit, SM clock, max SM clock:", card())
        ms, l2, T = time_kinds(args.batch, args.steps)
    print("shape: batch %d x %d samples, CM = %d" % (args.batch, T, args.cm))
    print("%-15s %4s %12s %12s %10s %10s %9s %10s" % ("kind", "n", "weight GB", "act GB", "HBM GB", "TFLOP", "ms",
                                                       "L2->SM GB/s"))
    tot = [0.0] * 4
    for n, name, w, a, hbm, f in kinds(args.batch, T, args.cm):
        t = ms.get(name)
        rate = "%10.0f" % ((w + a) / (t * 1e-3) / 1e9) if t else "%10s" % "-"
        print("%-15s %4d %12.2f %12.2f %10.2f %10.2f %9s %s" % (name, n, w / 1e9, a / 1e9, hbm / 1e9, f / 1e12,
                                                               "%.3f" % t if t else "-", rate))
        tot = [tot[0] + w, tot[1] + a, tot[2] + hbm, tot[3] + f]
    print("%-15s %4s %12.2f %12.2f %10.2f %10.2f" % ("total", "", tot[0] / 1e9, tot[1] / 1e9, tot[2] / 1e9,
                                                      tot[3] / 1e12))
    if l2 is not None:
        print("reference: torch sum over a 16 MB L2-resident buffer reads %.0f GB/s" % l2)


if __name__ == "__main__":
    main()
