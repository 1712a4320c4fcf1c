# -*- coding: utf-8 -*-
"""Time of the bf16 decoder's warm-up computed in parallel over time (wnb_decode_bf16_prefill) against its sequential
warm-up, and what it does to the first audio of a bf16 decode session.

    python tools/decode_bf16_prefill_times.py [--batches 1 8 64] [--reps 3] [--json out.json]

Shape: arctic 512/256 (256,28,512,256,10,3,2,80: rf 3 070, 80-sample frames, decode_math = "bf16"), with a one-sample
seed and with a 5 s seed (80 000 samples at 16 kHz).  For every (seed, B), each timed call sits between two synchronises
and the kernels are loaded by an untimed call first.  Reported (medians over --reps):
  * prefill: wnb_decode_bf16_prefill alone;
  * sequential warm-up: wnb_decode_bf16_at(pos0 = 0, max_n = 1) minus one free-running step
    (wnb_decode_bf16_at(pos0 = P - 1, max_n = 1) after a prefill); run once with the 5 s seed (about a minute per B);
  * first audio: creating a session and its first call (the prompt's frames and sample 0's), which runs the prefill.
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

CFG = (256, 28, 512, 256, 10, 3, 2, 80)
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
    """prefill(), step(pos0) -> closures over one batch's decode arguments (wnb_decode_bf16_at with max_n = 1)"""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import MODE_SAMPLING, _bf16_prefill, check, ptr, stream
    lib = _lib.load()
    B, T0 = x.shape
    Q, A, Ap, R, S, ks, U, L = (net.n_quantize, net.n_aux, net.n_aux_pad, net.n_resch, net.n_skipch, net.kernel_size,
                                net.upsampling_factor, len(net.dilations))
    P = max(T0, net.receptive_field)
    n_pad = P - T0
    w = net._decode_pack()
    wstream = net._decode_bf16_pack()
    upw = net.upsampling.conv.weight.detach().float().contiguous().view(-1)
    upb = net.upsampling.conv.bias.detach().float().contiguous().view(-1)
    dil = (ctypes.c_int32 * L)(*net.dilations)
    queues = torch.empty(lib.wnb_decode_bf16_workspace(B, R, ks, dil, L), dtype=torch.uint8, device="cuda")
    xs = torch.full((B, P + 1), Q // 2, dtype=torch.int32, device="cuda")
    xs[:, n_pad:P] = x.to(torch.int32)
    nsm = torch.ones(B, dtype=torch.int32, device="cuda")

    def prefill():
        _bf16_prefill(lib, xs, P, h, upw, upb, w, wstream, dil, L, queues, n_pad, A, Ap, R, S, ks, U)

    def step(pos0):
        check(lib.wnb_decode_bf16_at(ptr(xs), ptr(h), ptr(upw), ptr(upb), ptr(w["wf"]), ptr(w["bf"]), ptr(wstream), dil,
                                     L, ptr(queues), ptr(nsm), None, None, B, P, 1, n_pad, h.size(2), Q, A, Ap, R, S, ks,
                                     U, MODE_SAMPLING, ctypes.c_uint64(1), pos0, 0, 0, stream()), "decode_bf16_at")
    return prefill, step, P


def first_audio(net, x, h):
    """the prompt's frames have arrived; the first call gets them and the frame of sample 0"""
    F = (x.size(1) - 1) // net.upsampling_factor + 1

    def run():
        s = net.decode_session(x, [1000] * x.size(0), "sampling", seed=1)
        s.step(h[:, :, :F])
        assert max(s.last_counts) > 0
    return timed(run)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    name, q = card()
    print("card: %s, power limit: %s" % (name, q))
    rows = []
    with torch.no_grad():
        net = WaveNet(*CFG).cuda().eval()
        net.decode_math = "bf16"
        for sname, T0 in SEEDS.items():
            for B in args.batches:
                rng = np.random.RandomState(B)
                x = torch.from_numpy(rng.randint(0, 256, size=(B, T0))).cuda()
                h = torch.from_numpy(rng.standard_normal((B, CFG[1], (T0 + 1000) // CFG[-1] + 2))
                                     .astype(np.float32)).cuda()
                prefill, step, P = calls(net, x, h)
                prefill(); step(P - 1); first_audio(net, x, h)          # untimed: module load, allocations
                t_pre = [timed(prefill) for _ in range(args.reps)]
                t_free = []
                for _ in range(args.reps):
                    prefill()
                    t_free.append(timed(lambda: step(P - 1)))
                t_seq = [timed(lambda: step(0)) for _ in range(args.reps if T0 == 1 else 1)]
                t_first = [first_audio(net, x, h) for _ in range(args.reps)]
                row = {"seed": sname, "T0": T0, "B": B, "P": P, "prefill_ms": float(np.median(t_pre)) * 1e3,
                       "free_step_ms": float(np.median(t_free)) * 1e3,
                       "sequential_warmup_ms": (float(np.median(t_seq)) - float(np.median(t_free))) * 1e3,
                       "first_audio_s": float(np.median(t_first))}
                rows.append(row)
                print("%-14s B=%3d: prefill %8.2f ms, sequential warm-up %10.2f ms (%d steps), first audio %.4f s" % (
                    sname, B, row["prefill_ms"], row["sequential_warmup_ms"], P - 1, row["first_audio_s"]), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": q, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
