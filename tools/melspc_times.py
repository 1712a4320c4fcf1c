#!/usr/bin/env python
"""Timing of the melspc feature kernels (DESIGN.md §6 row f5): python tools/melspc_times.py [--reps R] [--out FILE]

For 64 synthetic 10 s int16 utterances at 16 kHz (hop 80, fftl 1024, 80 mels: the arctic recipes) and at 22.05 kHz
(hop 256: ljspeech): device time per stage by CUDA events (median of R launches after a warm-up), the float64 FLOPs and
algorithmic bytes of each stage from the shapes, the float64 restatement (tests/melspc_reference.py) on one host core
for one utterance, and bin/feature_extract.py end to end over the same 64 files on disk (a fresh process: interpreter
and torch start-up, wav reads, feature and wav writes included).  Prints the card name, power limit and SM clock beside
the numbers, and one JSON line."""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")          # the host restatement on one core
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
os.environ.setdefault("MKL_NUM_THREADS", "1")

import argparse  # noqa: E402
import json  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402
import tempfile  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorchwavenetvocoder_b200 import _lib  # noqa: E402
from pytorchwavenetvocoder_b200.utils import melspc as M  # noqa: E402
from tests import melspc_reference as R  # noqa: E402  (host baseline only)

CASES = [("arctic", 16000, 80, 5.0), ("ljspeech", 22050, 256, 11.61)]
FFTL, N_MELS, B, SECONDS, CUTOFF = 1024, 80, 64, 10, 70


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable"


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def signals(fs, seed=0):
    rng = np.random.RandomState(seed)
    n = SECONDS * fs
    t = np.arange(n) / fs
    out = []
    for i in range(B):
        f0 = 100 + 10 * i
        x = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 20)) * 2500 + rng.randn(n) * 300
        out.append(np.int16(np.clip(x, -32768, 32767)))
    return out


def stage_counts(lens, fs, hop):
    """float64 FLOPs and algorithmic bytes per stage.  FIR: 2 flops per tap and sample; reads int16, writes float64 (+
    int16 wav).  Frames: window 1, radix-2 FFT 10 flops per butterfly (fftl / 2 log2 fftl butterflies), |X| ~ 3 per bin,
    mel 2 per nonzero table entry; reads the float64 signal once, writes float32 features."""
    basis, lo, hi = M.mel_filterbank(fs, FFTL, N_MELS, 0, fs // 2)
    S = int(np.sum(lens))
    frames = int(np.sum(1 + np.asarray(lens) // hop))
    nb = FFTL // 2 + 1
    fir = {"gflop": 2.0 * M.N_TAPS * S / 1e9, "gb": (2 + 8 + 2) * S / 1e9}
    per_frame = FFTL + 10 * (FFTL // 2) * int(np.log2(FFTL)) + 3 * nb + 2 * int(np.sum(hi - lo))
    frm = {"gflop": per_frame * frames / 1e9, "gb": (8 * S + 4 * N_MELS * frames) / 1e9, "frames": frames,
           "flop_per_frame": per_frame}
    return fir, frm


def device_times(xs, fs, hop, reps):
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    flat = np.concatenate(xs)
    lens = np.array([len(x) for x in xs], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    foff = np.concatenate([[0], np.cumsum(1 + lens // hop)]).astype(np.int64)
    basis, lo, hi = M.mel_filterbank(fs, FFTL, N_MELS, 0, fs // 2)
    x = torch.from_numpy(flat).to(dev)
    offsets, frame_offsets = torch.from_numpy(off).to(dev), torch.from_numpy(foff).to(dev)
    taps = torch.from_numpy(M.lowcut_taps(fs, CUTOFF)).to(dev)
    y = torch.empty(len(flat), dtype=torch.float64, device=dev)
    y16 = torch.empty(len(flat), dtype=torch.int16, device=dev)
    window = torch.from_numpy(M.hann_window(FFTL)).to(dev)
    tw = torch.from_numpy(np.array(M.fft_twiddles(FFTL))).to(dev)
    mel = torch.from_numpy(np.array(basis)).to(dev)
    mlo, mhi = torch.from_numpy(np.array(lo)).to(dev), torch.from_numpy(np.array(hi)).to(dev)
    out = torch.empty(int(foff[-1]), N_MELS, dtype=torch.float32, device=dev)
    p = _lib.ptr

    def lowcut():
        _lib.check(lib.wnb_melspc_lowcut(p(x), 1, p(offsets), B, int(lens.max()), p(taps), M.N_TAPS, p(y), p(y16),
                                         _lib.stream()), "melspc_lowcut")

    def frames():
        _lib.check(lib.wnb_melspc(p(y), 0, p(offsets), p(frame_offsets), B, int(foff[-1]), FFTL, hop, p(window), p(tw),
                                  p(mel), p(mlo), p(mhi), N_MELS, p(out), _lib.stream()), "melspc")

    for _ in range(3):
        lowcut()
        frames()
    torch.cuda.synchronize()
    t_fir = median_ms(lowcut, reps)
    t_frm = median_ms(frames, reps)
    t_both = median_ms(lambda: (lowcut(), frames()), reps)
    return t_fir, t_frm, t_both, lens


def cli_end_to_end(xs, fs, shiftms):
    from scipy.io import wavfile
    with tempfile.TemporaryDirectory() as d:
        wd = os.path.join(d, "wav")
        os.makedirs(wd)
        for i, x in enumerate(xs):
            wavfile.write(os.path.join(wd, "u%02d.wav" % i), fs, x)
        cmd = [sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.feature_extract", "--waveforms", wd, "--wavdir",
               os.path.join(d, "wav_hpf"), "--hdf5dir", os.path.join(d, "hdf5"), "--feature_type", "melspc", "--fs",
               str(fs), "--shiftms", str(shiftms), "--mspc_dim", str(N_MELS), "--highpass_cutoff", str(CUTOFF),
               "--fftl", str(FFTL), "--fmin", "", "--fmax", "", "--batch_size", str(B), "--verbose", "0"]
        t0 = time.time()
        r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT)
        wall = time.time() - t0
        if r.returncode != 0:
            raise RuntimeError(r.stdout.decode()[-2000:])
        t0 = time.time()
        subprocess.run([sys.executable, "-c", "import torch, pytorchwavenetvocoder_b200.utils.melspc"], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), check=True)
        startup = time.time() - t0
        n_out = len(os.listdir(os.path.join(d, "hdf5")))
    return wall, startup, n_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-cli", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("melspc_times.py measures the GPU kernels and needs a GPU")
    torch.cuda.set_device(0)
    info = {"card": card(), "rows": []}
    print("card (name, power limit, SM clock, max SM clock):", info["card"])
    for name, fs, hop, shiftms in CASES:
        xs = signals(fs)
        t_fir, t_frm, t_both, lens = device_times(xs, fs, hop, a.reps)
        fir, frm = stage_counts(lens, fs, hop)
        t0 = time.time()
        R.melspc(xs[0], fs, FFTL, hop, N_MELS, taps=M.lowcut_taps(fs, CUTOFF))
        host_s = time.time() - t0
        row = {"case": name, "fs": fs, "hop": hop, "fftl": FFTL, "utterances": B, "samples": int(np.sum(lens)),
               "frames": frm["frames"],
               "lowcut_ms": t_fir[0], "lowcut_ms_min_max": t_fir[1:], "lowcut_gflop": fir["gflop"],
               "lowcut_gb": fir["gb"], "lowcut_fp64_tflops": fir["gflop"] / t_fir[0],
               "frames_ms": t_frm[0], "frames_ms_min_max": t_frm[1:], "frames_gflop": frm["gflop"],
               "frames_gb": frm["gb"], "frames_fp64_tflops": frm["gflop"] / t_frm[0],
               "flop_per_frame": frm["flop_per_frame"], "both_ms": t_both[0],
               "host_oracle_s_per_utterance_1core": host_s, "host_oracle_s_for_batch_1core_est": host_s * B}
        if not a.no_cli:
            wall, startup, n_out = cli_end_to_end(xs, fs, shiftms)
            row.update({"cli_wall_s": wall, "cli_process_startup_s": startup, "cli_files_written": n_out})
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
