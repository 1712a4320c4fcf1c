#!/usr/bin/env python
"""Timing of the device-resident corpus (DESIGN.md §6 row f9): python tools/corpus_times.py [--hours 1,24] [--steps K]

1. Preparation (``utils/corpus.prepare_corpus``) of seeded synthetic corpora of 10 s int16 wavs written to a temporary
   directory: arctic settings (16 kHz, hop 80, 80 mels, mcep order 24) and ljspeech settings (22.05 kHz, hop 256, 80
   mels, order 35), with and without noise shaping, split per stage (wav reads, low-cut + mel-spectrogram + resident
   copies, mcep, host statistics, MLSA), for each size in --hours (the largest only at 16 kHz with noise shaping).
2. ``wnb_make_train_batch_corpus`` alone at the BASELINE batch (8 x 23 040 samples, 28 aux dims) by CUDA events, beside
   ``wnb_make_train_batch`` (the ring loader's kernel) at the same shape.
3. The BASELINE training step (bench.py's model and Adam, tf32) fed by ``DeviceCorpusGenerator`` over a 1 h corpus
   against ``DeviceTrainGenerator`` reading the same corpus's low-cut wavs and feature files, alternated three times in
   this process; ms per step including the generator call, device-synchronised.
Prints the card name, power limit and SM clock beside the numbers, and one JSON line."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorchwavenetvocoder_b200 import _lib  # noqa: E402
from pytorchwavenetvocoder_b200.utils import write_wav_int16  # noqa: E402
from pytorchwavenetvocoder_b200.utils.corpus import prepare_corpus  # noqa: E402

SETTINGS = {"arctic": dict(fs=16000, shiftms=5.0, mcep_dim=24), "ljspeech": dict(fs=22050, shiftms=11.61, mcep_dim=35)}
SECONDS = 10
CFG = (256, 28, 64, 512, 10, 3, 2, 80)       # bench.py's BASELINE shape
BATCH, BATCH_LENGTH = 8, 20000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable"


def write_corpus(root, fs, hours, seed):
    """seeded speech-like wavs of 10 s +- 20 %: slices of one 2-minute signal (harmonic tones with a moving f0, and
    noise) at random offsets"""
    os.makedirs(root)
    rng = np.random.RandomState(seed)
    t = np.arange(120 * fs) / fs
    ph = 2 * np.pi * np.cumsum(100 + 60 * np.sin(2 * np.pi * t / 1.3)) / fs
    base = np.int16(np.clip(sum(np.sin(k * ph) / k for k in range(1, 6)) * 0.2 + 0.01 * rng.standard_normal(len(t)),
                            -1, 1) * 30000)
    names, total, i = [], 0, 0
    while total < hours * 3600 * fs:
        n = int(SECONDS * fs * rng.uniform(0.8, 1.2))
        o = rng.randint(0, len(base) - n)
        p = os.path.join(root, "s%05d.wav" % i)
        write_wav_int16(p, fs, base[o:o + n])
        names.append(p)
        total += n
        i += 1
    return names, total


def prep_case(tmp, name, hours, ns, n_mels=80, seed=0):
    s = SETTINGS[name]
    root = os.path.join(tmp, "%s_%gh" % (name, hours))
    if not os.path.exists(root):
        write_corpus(root, s["fs"], hours, seed)
    wavs = sorted(os.path.join(root, f) for f in os.listdir(root))
    torch.cuda.synchronize()
    t0 = time.time()
    c = prepare_corpus(wavs, fs=s["fs"], shiftms=s["shiftms"], fftl=1024, mspc_dim=n_mels, highpass_cutoff=70,
                       noise_shaping=ns, mcep_dim=s["mcep_dim"], mcep_alpha=0.41, mag=0.5)
    torch.cuda.synchronize()
    total = time.time() - t0
    row = dict(corpus=name, hours=hours, noise_shaping=ns, utterances=len(wavs), samples=int(c.wave.numel()),
               frames=int(c.feat.size(0)), resident_gb=round((2 * c.wave.numel() + 4 * c.feat.numel()) / 1e9, 3),
               total_s=round(total, 2), **{k + "_s": round(v, 3) for k, v in c.times.items()})
    print("prepare %-8s %5g h %-5s: %d utts, %.2f GB resident, %.2f s  (%s)" % (
        name, hours, "ns" if ns else "plain", len(wavs), row["resident_gb"], total,
        ", ".join("%s %.2f" % kv for kv in c.times.items())), flush=True)
    return row, c, wavs


def median_ms(fn, reps, inner):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / inner)
    return round(float(np.median(ts)), 4)


def kernel_times(corpus):
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceCorpusGenerator
    lib, P = _lib.load(), _lib.ptr
    rf = 1 + (CFG[6] - 1) * sum([2 ** i for i in range(CFG[4])] * CFG[5])
    g = DeviceCorpusGenerator(corpus, rf, BATCH_LENGTH, BATCH)
    g.next()
    B, T, Tf, D = g.B, g.T, g.Tf, g.D
    x = torch.empty(B, T, dtype=torch.int64, device="cuda")
    t = torch.empty_like(x)
    h = torch.empty(B, D, Tf, dtype=torch.float32, device="cuda")
    mean = torch.zeros(D, dtype=torch.float64, device="cuda")
    scale = torch.ones(D, dtype=torch.float64, device="cuda")
    tab, (b0, b1) = g.table, g.table_span

    def corpus_batch():
        lib.wnb_make_train_batch_corpus(P(corpus.wave), P(corpus.feat), P(tab[0]), P(tab[1]), tab.size(1), b0, b1, b0,
                                        g.hop, g.U, P(mean), P(scale), P(x), P(t), P(h), B, T, Tf, D, g.feat_f64, 256,
                                        _lib.stream())
    cap_s = 1 << 22
    wave = torch.zeros(cap_s, dtype=torch.float32, device="cuda")
    feat = torch.zeros(cap_s // g.U + 256, D, dtype=torch.float32, device="cuda")

    def ring_batch():
        lib.wnb_make_train_batch(P(wave), P(feat), None, 0, g.hop, g.U, cap_s, feat.size(0), P(mean), P(scale), P(x),
                                 P(t), P(h), B, T, Tf, D, g.feat_f64, 256, _lib.stream())
    for fn in (corpus_batch, ring_batch):
        fn()
    torch.cuda.synchronize()
    res = dict(B=B, T=T, D=D, table_utterances=int(tab.size(1)), corpus_kernel_ms=median_ms(corpus_batch, 7, 50),
               ring_kernel_ms=median_ms(ring_batch, 7, 50))
    print("batch kernel (B %d, T %d, D %d, table of %d utterances): corpus %.4f ms, ring %.4f ms" % (
        B, T, D, res["table_utterances"], res["corpus_kernel_ms"], res["ring_kernel_ms"]), flush=True)
    return res


def step_times(tmp, steps):
    """the BASELINE step fed by the resident corpus and by DeviceTrainGenerator from files, alternated"""
    from pytorchwavenetvocoder_b200.bin import feature_extract
    from pytorchwavenetvocoder_b200.nets import WaveNet, initialize
    from pytorchwavenetvocoder_b200.optim import Adam
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceCorpusGenerator, DeviceTrainGenerator
    _, corpus, wavs = prep_case(tmp, "arctic", 1, False, n_mels=CFG[1])
    scp = os.path.join(tmp, "steps.scp")
    open(scp, "w").write("\n".join(wavs) + "\n")
    hdf5, hpf = os.path.join(tmp, "steps_hdf5"), os.path.join(tmp, "steps_hpf")
    feature_extract.main(["--waveforms", scp, "--hdf5dir", hdf5, "--wavdir", hpf, "--feature_type", "melspc",
                          "--mspc_dim", str(CFG[1]), "--verbose", "0"])
    feats = sorted(os.path.join(hdf5, f) for f in os.listdir(hdf5))
    hpf_wavs = sorted(os.path.join(hpf, f) for f in os.listdir(hpf))
    torch.manual_seed(20260924)
    net = WaveNet(*CFG)
    net.apply(initialize)
    net.math_mode = "tf32"
    net = net.cuda().train()
    opt = Adam(net.parameters(), lr=1e-4, module=net)
    rf = net.receptive_field
    np.random.seed(1)
    gens = {"corpus": DeviceCorpusGenerator(corpus, rf, BATCH_LENGTH, BATCH, mean=corpus.mean, scale=corpus.scale),
            "files": DeviceTrainGenerator(hpf_wavs, feats, rf, BATCH_LENGTH, BATCH, feature_type="melspc",
                                          mean=corpus.mean, scale=corpus.scale, upsampling_factor=corpus.U)}

    def run(gen, n):
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(n):
            (x, h), t = gen.next()
            loss = net.forward_loss(x, h, t, rf)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
        torch.cuda.synchronize()
        return (time.time() - t0) * 1e3 / n
    for g in gens.values():
        run(g, 5)                                    # warm-up: modules, allocator, reader threads
    res = {k: [] for k in gens}
    for _ in range(3):
        for k, g in gens.items():
            res[k].append(round(run(g, steps), 3))
    out = {"step_ms_" + k: float(np.median(v)) for k, v in res.items()}
    out.update({"step_ms_runs_" + k: v for k, v in res.items()})
    print("BASELINE step (8 x 23 040, tf32): resident corpus %.3f ms, files %.3f ms (runs %s / %s)" % (
        out["step_ms_corpus"], out["step_ms_files"], res["corpus"], res["files"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hours", default="1,24", help="corpus sizes in hours; the largest runs at 16 kHz with noise "
                                                   "shaping only")
    ap.add_argument("--steps", default=30, type=int, help="training steps per alternated run")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("corpus_times.py measures on a GPU; none is visible")
    hours = sorted(float(h) for h in args.hours.split(","))
    name = card()
    print("card: %s" % name, flush=True)
    tmp = tempfile.mkdtemp(prefix="corpus_times_")
    try:
        rows = []
        for hh in hours:
            cases = [("arctic", True)] if (hh == hours[-1] and len(hours) > 1) else [
                (c, ns) for c in SETTINGS for ns in (False, True)]
            for corpus_name, ns in cases:
                row, c, _ = prep_case(tmp, corpus_name, hh, ns)
                rows.append(row)
                del c
                torch.cuda.empty_cache()
            for corpus_name in SETTINGS:
                shutil.rmtree(os.path.join(tmp, "%s_%gh" % (corpus_name, hh)), ignore_errors=True)
        _, c, _ = prep_case(tmp, "arctic", hours[0], False, n_mels=CFG[1])
        kern = kernel_times(c)
        del c
        torch.cuda.empty_cache()
        steps = step_times(tmp, args.steps)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(dict(card=name, prepare=rows, kernel=kern, steps=steps))
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
