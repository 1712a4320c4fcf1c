# -*- coding: utf-8 -*-
"""Timing of mel-cepstral distortion (DESIGN.md §6 row f8) at arctic settings: 10 s utterances (1 988 frames of order
24, fs 16 000, 5 ms, fftl 1 024, alpha 0.41), decoded side = the natural wav plus white noise.

- ``mcd_batch`` for 1, 8 and 64 pairs, aligned and DTW: the kernel alone (CUDA events around the library launch, inputs
  already on the device, median of repeated launches) and the whole call (host clock; it ends in the copy back, a device
  synchronise), medians;
- the float64 restatement (tests/distortion_reference.py) of one pair on one host core;
- the whole CLI (``bin/calc_mcd.py``, a fresh process: imports, wav reading, mcep analysis, MCD, TSV) on 64 pairs;
- the card name and its power limit, printed in the same run.

    python tools/mcd_times.py [--reps 10] [--out DIR]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pytorchwavenetvocoder_b200._lib import check, load, ptr, stream  # noqa: E402
from pytorchwavenetvocoder_b200.utils import distortion as DI  # noqa: E402
from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch  # noqa: E402
from tests import distortion_reference as R  # noqa: E402

FS, FFTL, HOP, ORDER, ALPHA = 16000, 1024, 80, 24, 0.41


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _speechlike(rng, n, amp=8000.0):
    from scipy.signal import lfilter
    e = rng.randn(n) * 300.0
    e[::int(rng.randint(60, 140))] += amp
    y = lfilter([1.0], [1.0, -1.4, 0.75, -0.15], e)
    return np.int16(y / (np.abs(y).max() + 1e-9) * amp)


def kernel_ms(refs, decs, dtw, reps):
    """Median CUDA-event time of one library launch over the pairs, inputs on the device."""
    dev = torch.device("cuda", 0)
    n, cols = len(refs), refs[0].shape[1]
    roff = np.concatenate([[0], np.cumsum([len(a) for a in refs])]).astype(np.int64)
    doff = np.concatenate([[0], np.cumsum([len(b) for b in decs])]).astype(np.int64)
    r, d = torch.from_numpy(np.concatenate(refs)).to(dev), torch.from_numpy(np.concatenate(decs)).to(dev)
    ro, do = torch.from_numpy(roff).to(dev), torch.from_numpy(doff).to(dev)
    sums = torch.empty(n, dtype=torch.float64, device=dev)
    counts = torch.empty(n, dtype=torch.int64, device=dev)
    need = sum(DI.dtw_workspace_bytes(len(a), len(b)) for a, b in zip(refs, decs))
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=dev)
    lib = load()

    def launch():
        if dtw:
            check(lib.wnb_mcd_dtw(ptr(r), ptr(d), cols, ptr(ro), ptr(do), roff.ctypes.data, doff.ctypes.data, n,
                                  ptr(ws), need, ptr(sums), ptr(counts), None, stream()), "mcd_dtw")
        else:
            check(lib.wnb_mcd_aligned(ptr(r), ptr(d), cols, ptr(ro), ptr(do), roff.ctypes.data, doff.ctypes.data, n,
                                      ptr(sums), ptr(counts), stream()), "mcd_aligned")
    for _ in range(2):
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
    return float(np.median(ms)), need


def call_ms(refs, decs, dtw, reps):
    DI.mcd_batch(refs, decs, dtw=dtw)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        DI.mcd_batch(refs, decs, dtw=dtw)
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the CLI's wavs and TSV (default: a temporary one)")
    args = ap.parse_args()
    print("card: %s" % card())
    rng = np.random.RandomState(0)
    nat = [_speechlike(rng, 10 * FS) for _ in range(64)]
    dec = [np.int16(np.clip(x + rng.randn(len(x)) * 300, -32768, 32767)) for x in nat]
    t0 = time.perf_counter()
    R_frames = mcep_batch(nat, FS, FFTL, HOP, ORDER, ALPHA, highpass_cutoff=70)
    D_frames = mcep_batch(dec, FS, FFTL, HOP, ORDER, ALPHA, highpass_cutoff=70)
    print("mcep of 2 x 64 x 10 s: %.0f ms (%d frames per utterance, order %d)"
          % ((time.perf_counter() - t0) * 1e3, len(R_frames[0]), ORDER))
    for n in (1, 8, 64):
        for dtw in (False, True):
            k, need = kernel_ms(R_frames[:n], D_frames[:n], dtw, args.reps)
            c = call_ms(R_frames[:n], D_frames[:n], dtw, args.reps)
            print("%2d pairs %-7s: kernel %8.3f ms, mcd_batch %8.3f ms%s"
                  % (n, "dtw" if dtw else "aligned", k, c, ", workspace %.1f MB" % (need / 2 ** 20) if dtw else ""))
    got = DI.mcd_batch(R_frames[:1], D_frames[:1], dtw=True, return_path=True)
    t0 = time.perf_counter()
    s, path = R.dtw(R_frames[0], D_frames[0])
    dtw_ref = time.perf_counter() - t0
    t0 = time.perf_counter()
    s_al, _ = R.aligned(R_frames[0], D_frames[0])
    al_ref = time.perf_counter() - t0
    assert got.sums[0] == s and np.array_equal(got.paths[0], path)
    assert DI.mcd_batch(R_frames[:1], D_frames[:1]).sums[0] == s_al
    print("float64 restatement, one pair on one host core: dtw %.0f ms, aligned %.2f ms (device results equal it bit "
          "for bit); one pair's MCD %.3f dB aligned, %.3f dB along %d DTW steps"
          % (dtw_ref * 1e3, al_ref * 1e3, DI.K * s_al / len(R_frames[0]), DI.K * s / len(path), len(path)))
    with tempfile.TemporaryDirectory() as tmp:
        base = args.out or tmp
        from scipy.io import wavfile
        for side, xs in (("nat", nat), ("dec", dec)):
            os.makedirs(os.path.join(base, side), exist_ok=True)
            for k, x in enumerate(xs):
                wavfile.write(os.path.join(base, side, "u%02d.wav" % k), FS, x)
        for extra in ([], ["--dtw"]):
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.calc_mcd", "--reference",
                                os.path.join(base, "nat"), "--decoded", os.path.join(base, "dec"), "--outfile",
                                os.path.join(base, "mcd%s.tsv" % "".join(extra))] + extra, cwd=ROOT,
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
            wall = time.perf_counter() - t0
            last = [line for line in r.stdout.decode().splitlines() if "corpus MCD" in line]
            print("CLI on 64 pairs%s: exit %d, %.2f s wall; %s" % (" --dtw" if extra else "", r.returncode, wall,
                                                                   last[-1].split(": ", 1)[-1] if last else "?"))


if __name__ == "__main__":
    main()
