#!/usr/bin/env python
"""Timing of streaming mel-spectrogram extraction (DESIGN.md §6 row f7): python tools/melspc_stream_times.py [--out FILE]

Cases: arctic (16 kHz, fftl 1024, hop 80, 80 mels, cutoff 70) and ljspeech (22.05 kHz, fftl 1024, hop 256, 80 mels,
cutoff 70), synthetic 10 s int16 signals.  Rows, each by CUDA events over many calls after a warm-up:
* ``MelspcStream.push`` per call for 1 / 8 / 64 keys, with one-hop chunks and with 1 600-sample chunks (host planning,
  the segment-table copy and both launches included);
* whole-file ``melspc_batch`` over the same keys' 10 s signals (host copies included);
* arctic only: one push of one-hop chunks next to one bf16 decode-session step of one frame for as many rows, at the
  arctic-melspc shape 256,80,512,256,10,3,2,80.
Prints the card name, power limit and SM clock beside the numbers, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorchwavenetvocoder_b200.utils import melspc as M  # noqa: E402

CASES = [("arctic", 16000, 80), ("ljspeech", 22050, 256)]
FFTL, N_MELS, CUTOFF, SECONDS = 1024, 80, 70, 10
ARCTIC_MELSPC = (256, 80, 512, 256, 10, 3, 2, 80)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable"


def per_call_ms(fn, calls, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def signals(fs, n_keys, seed=0):
    rng = np.random.RandomState(seed)
    t = np.arange(SECONDS * fs) / fs
    return [np.int16(np.clip(sum(np.sin(2 * np.pi * (100 + 10 * i) * h * t) / h for h in range(1, 12)) * 2500
                             + rng.randn(len(t)) * 300, -32768, 32767)) for i in range(n_keys)]


def push_ms(fs, hop, xs, chunk):
    s = M.MelspcStream(fs, FFTL, hop, N_MELS, highpass_cutoff=CUTOFF)
    dev = [torch.from_numpy(x).cuda() for x in xs]
    pos = [0]
    calls = min(200, (len(xs[0]) - FFTL) // chunk - 10)

    def one():
        p = pos[0]
        s.push({k: d[p:p + chunk] for k, d in enumerate(dev)})
        pos[0] = p + chunk
    return per_call_ms(one, calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("melspc_stream_times.py measures the GPU kernels and needs a GPU")
    torch.cuda.set_device(0)
    info = {"card": card(), "rows": []}
    print("card (name, power limit, SM clock, max SM clock):", info["card"])
    for name, fs, hop in CASES:
        all_xs = signals(fs, 64)
        for keys in (1, 8, 64):
            xs = all_xs[:keys]
            row = {"case": name, "fs": fs, "hop": hop, "keys": keys,
                   "push_ms_hop_chunks": push_ms(fs, hop, xs, hop),
                   "push_ms_1600_chunks": push_ms(fs, hop, xs, 1600),
                   "melspc_batch_ms_10s": per_call_ms(
                       lambda: M.melspc_batch(xs, fs, FFTL, hop, N_MELS, highpass_cutoff=CUTOFF), 5, 2)}
            info["rows"].append(row)
            print(json.dumps(row))
    from oracle import wavenet_oracle as O
    from tests.util import our_model
    cfg = O.Config(*ARCTIC_MELSPC)
    net = our_model(cfg, O.make_params(cfg, 1)).eval()
    net.decode_math = "bf16"
    for keys in (1, 8, 64):
        x = torch.full((keys, 1), 128, dtype=torch.long, device="cuda")
        with torch.no_grad():
            sess = net.decode_session(x, [80 * 400 - 1] * keys)
            h = torch.zeros(keys, N_MELS, 1, device="cuda")
            sess.step(torch.zeros(keys, N_MELS, 2, device="cuda"))
            step = per_call_ms(lambda: sess.step(h), 100)
        row = {"case": "arctic push vs bf16 decode step", "keys": keys,
               "push_ms_hop_chunks": push_ms(16000, 80, signals(16000, keys), 80), "decode_step_ms_one_frame": step}
        info["rows"].append(row)
        print(json.dumps(row))
    line = json.dumps(info)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
