# -*- coding: utf-8 -*-
"""Timing of the STFT mel-cepstrum kernel (DESIGN.md §6 row f6) for the arctic and ljspeech batch shapes, 64 utterances
of 10 s each, with the low-cut filter excluded:

- the kernel time (CUDA events around wnb_mcep alone, after warm-up, median of repeated launches);
- the float64 FLOPs from the shapes and the measured update counts (FFT 5 L log2 L; initial value 2 (M + 2) (L/2 + 1);
  per iteration 2 M + 6 for Clenshaw and R_k per bin, 4 (2M + 1) per bin for r, (M + 1)^3 / 3 + 2 (M + 1)^2 for the
  solve, plus one more evaluation of r for the convergence test that stops);
- the histogram of the update counts;
- the oracle (oracle/mcep_oracle.c, one host core) per frame, on a sample of frames;
- the card name and its power limit, printed in the same run.

    python tools/mcep_times.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import mcep_oracle as MO  # noqa: E402
from pytorchwavenetvocoder_b200._lib import check, load, ptr, stream  # noqa: E402
from pytorchwavenetvocoder_b200.utils import mcep as MC  # noqa: E402
from pytorchwavenetvocoder_b200.utils.melspc import fft_twiddles  # noqa: E402

SHAPES = {"arctic": dict(fs=16000, fftl=1024, hop=80, order=25, alpha=0.41),
          "ljspeech": dict(fs=22050, fftl=1024, hop=256, order=35, alpha=0.455)}


def _speechlike(rng, n, amp=8000.0):
    from scipy.signal import lfilter
    e = rng.randn(n) * 300.0
    e[::int(rng.randint(60, 140))] += amp
    y = lfilter([1.0], [1.0, -1.4, 0.75, -0.15], e)
    return np.int16(y / (np.abs(y).max() + 1e-9) * amp)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def run(name, cfg, reps):
    rng = np.random.RandomState(0)
    fs, L, hop, M, a = cfg["fs"], cfg["fftl"], cfg["hop"], cfg["order"], cfg["alpha"]
    xs = [_speechlike(rng, 10 * fs) for _ in range(64)]
    lens = np.array([len(x) for x in xs], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(lens)])
    foff = np.concatenate([[0], np.cumsum((lens - L) // hop + 1)])
    nf = int(foff[-1])
    dev = torch.device("cuda", 0)
    t = lambda a_: torch.from_numpy(np.ascontiguousarray(a_)).to(dev)  # noqa: E731
    x, o, fo = t(np.concatenate(xs)), t(off), t(foff)
    win, tw, cw = t(MC.hamming_window(L)), t(np.array(fft_twiddles(L))), t(MC.warped_cos(L, a))
    W, al = t(np.array(MC.init_map(L, M, a))), t(MC.neg_alpha_powers(M, a))
    out = torch.empty(nf, M + 1, dtype=torch.float32, device=dev)
    its = torch.empty(nf, dtype=torch.int32, device=dev)

    def launch():
        check(load().wnb_mcep(ptr(x), 1, ptr(o), ptr(fo), 64, nf, L, hop, M, a, ptr(win), ptr(tw), ptr(cw), ptr(W),
                              ptr(al), 2, 30, 1e-3, MC.EPS, MC.MIN_DET, ptr(out), ptr(its), stream()), "mcep")
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    med = float(np.median(ms))
    n = its.cpu().numpy().astype(np.int64)
    nb = L // 2 + 1
    per_iter = nb * (2 * M + 6) + nb * 4 * (2 * M + 1) + (M + 1) ** 3 / 3.0 + 2 * (M + 1) ** 2
    flops = nf * (5 * L * np.log2(L) + 2 * (M + 2) * nb) + (n.sum() + nf) * per_iter
    hist = np.bincount(n, minlength=1)
    sample = MO.frames(xs[0], L, hop)[:200]
    t0 = time.perf_counter()
    for f in sample:
        MO.mcep(f, M, a)
    oracle_ms = (time.perf_counter() - t0) / len(sample) * 1e3
    print("%s: 64 x %d samples, %d frames, fftl %d, order %d, alpha %g" % (name, 10 * fs, nf, L, M, a))
    print("  kernel: median %.3f ms over %d launches (min %.3f, max %.3f)" % (med, reps, min(ms), max(ms)))
    print("  FLOPs (float64): %.3g, %.2f TFLOP/s; mean updates per frame %.3f" % (flops, flops / med * 1e-9, n.mean()))
    print("  update counts: %s" % {i: int(c) for i, c in enumerate(hist) if c})
    print("  oracle on one host core: %.3f ms per frame, %.1f s for the batch (extrapolated)"
          % (oracle_ms, oracle_ms * nf * 1e-3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    print("card: %s" % card())
    for name, cfg in SHAPES.items():
        run(name, cfg, args.reps)


if __name__ == "__main__":
    main()
