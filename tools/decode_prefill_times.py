# -*- coding: utf-8 -*-
"""Time of the decode warm-up computed in parallel over time (wnb_decode_warp_prefill) against the sequential warm-up,
and what it does to the first audio of a decode session.

    python tools/decode_prefill_times.py [--batches 1 8 64] [--reps 5] [--json out.json]

Shape: the BASELINE 64/512 model (fp32 warp-tiled decoder, rf 3 070, 80-sample frames), with a one-sample seed and with a
5 s seed (80 000 samples at 16 kHz).  For every (seed, B), each timed call sits between two synchronises and every shape
is run once untimed first.  Reported (medians over --reps):
  * prefill: wnb_decode_warp_prefill alone;
  * sequential warm-up: wnb_decode_warp_at(pos0 = 0, max_n = 1) minus one free-running step
    (wnb_decode_warp_at(pos0 = P - 1, max_n = 1) after a prefill);
  * first audio: creating a session and its first 1-frame call, which now runs the prefill.
Prints the card and its power limit, read in the same run."""
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

CFG = (256, 28, 64, 512, 10, 3, 2, 80)
SEEDS = {"1-sample seed": 1, "5 s seed": 80000}


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


def calls(net, x, h):
    """prefill(), step(pos0) -> closures over one batch's decode arguments (wnb_decode_warp_at with max_n = 1)"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import MODE_SAMPLING, _warp_prefill, check, ptr, stream
    lib = _lib.load()
    B, T0 = x.shape
    L, A, U = len(net.dilations), net.n_aux, net.upsampling_factor
    P = max(T0, net.receptive_field)
    n_pad = P - T0
    w = net._decode_pack()
    W, CL = lib.wnb_decode_warp_plan(B), lib.wnb_decode_warp_cluster(B)
    wstream = net._decode_warp_pack(W, CL)
    upw = net.upsampling.conv.weight.detach().float().contiguous().view(-1)
    upb = net.upsampling.conv.bias.detach().float().contiguous().view(-1)
    dil = (ctypes.c_int32 * L)(*net.dilations)
    queues = torch.empty(lib.wnb_decode_workspace(B, 64, 2, dil, L) // 4, device="cuda")
    xs = torch.full((B, P + 1), 128, dtype=torch.int32, device="cuda")
    xs[:, n_pad:P] = x.to(torch.int32)
    nsm = torch.ones(B, dtype=torch.int32, device="cuda")

    def prefill():
        _warp_prefill(lib, xs, P, h, upw, upb, w, dil, L, queues, n_pad, A, U, CL)

    def step(pos0):
        check(lib.wnb_decode_warp_at(ptr(xs), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]), ptr(wstream),
                                     ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), dil, L, ptr(queues),
                                     ptr(nsm), None, None, B, P, 1, n_pad, h.size(2), A, U, MODE_SAMPLING,
                                     ctypes.c_uint64(1), W, CL, pos0, 0, 0, stream()), "decode_warp_at")
    return prefill, step, P


def first_audio(net, x, h, P):
    """the prompt's frames have arrived; the first call gets them and the frame of sample 0"""
    U = net.upsampling_factor
    F = (x.size(1) - 1) // U + 1

    def run():
        s = net.decode_session(x, [1000] * x.size(0), "sampling", seed=1)
        s.step(h[:, :, :F])
        assert max(s.last_counts) > 0
    return timed(run)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    name, q = card()
    print("card: %s, power limit: %s" % (name, q))
    rows = []
    with torch.no_grad():
        net = WaveNet(*CFG).cuda().eval()
        for sname, T0 in SEEDS.items():
            for B in args.batches:
                rng = np.random.RandomState(B)
                x = torch.from_numpy(rng.randint(0, 256, size=(B, T0))).cuda()
                h = torch.from_numpy(rng.standard_normal((B, CFG[1], (T0 + 1000) // CFG[-1] + 2))
                                     .astype(np.float32)).cuda()
                prefill, step, P = calls(net, x, h)
                prefill(); step(P - 1); step(0); first_audio(net, x, h, P)          # untimed: module load, allocations
                t_pre = [timed(prefill) for _ in range(args.reps)]
                t_free = []
                for _ in range(args.reps):
                    prefill()
                    t_free.append(timed(lambda: step(P - 1)))
                t_seq = [timed(lambda: step(0)) for _ in range(max(1, args.reps if T0 == 1 else 2))]
                t_first = [first_audio(net, x, h, P) for _ in range(args.reps)]
                row = {"seed": sname, "T0": T0, "B": B, "P": P, "prefill_ms": float(np.median(t_pre)) * 1e3,
                       "free_step_ms": float(np.median(t_free)) * 1e3,
                       "sequential_warmup_ms": (float(np.median(t_seq)) - float(np.median(t_free))) * 1e3,
                       "first_audio_s": float(np.median(t_first))}
                rows.append(row)
                print("%-14s B=%3d: prefill %8.2f ms, sequential warm-up %9.2f ms (%d steps), first audio %.4f s" % (
                    sname, B, row["prefill_ms"], row["sequential_warmup_ms"], P - 1, row["first_audio_s"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": q, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
