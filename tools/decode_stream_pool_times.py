# -*- coding: utf-8 -*-
"""The streaming decoder's parallel warm-up (wnb_decode_stream_prefill) and its decode pools, timed.

    python tools/decode_stream_pool_times.py [--json out.json] [--no-sequential] [--parts abcde]

Shapes: arctic fp32 (256,28,512,256,10,3,2,80: 30 layers, rf 3 070) and ljspeech-melspc fp32 (256,80,512,256,10,3,3,256:
ks 3, rf 6 139), random weights, Philox sampling.  Every timed region ends in a synchronise, after an untimed run of the
same shape.  Reported:
  a. the prefill against the sequential warm-up (wnb_decode_stream_at from pos0 = 0 with max_n = 1, so one decoded
     step rides along) at B = 1, 8 and 64, for a one-sample seed and a 5 s prompt (the prefill only: the
     sequential warm-up over a 5 s prompt is P - 1 steps and is not run), with the prefill's FLOPs from shapes,
     2 * sum_l window(l + 1) * (K1 * 2R + R * R), and its achieved rate;
  b. first audio of a B = 1 decode session: the first step(), fed 2 frames, until its codes are on the host;
  c. arctic B = 64: one full kernel="stream" pool call of 480 steps against DecodeSession.step of 480 samples;
  d. admission (prefill + one wnb_decode_pool_move + a 1-step call) of 1, 8 and 64 streams, against a 1-step call;
  e. (--parts e) short warm-ups: the prefill and the sequential warm-up against the number of warm-up positions P - 1
     (15 .. 1 023), at three small models and B = 1, 5 and 64, median of 5 runs each.
Prints the card, its power limit and its SM clock, read in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"arctic": ((256, 28, 512, 256, 10, 3, 2, 80), 16000), "ljspeech_melspc": ((256, 80, 512, 256, 10, 3, 3, 256),
                                                                                    22050)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=20).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    parts = [p.strip() for p in q.split(",")] if q else []
    return name, parts[0] if parts else "unavailable", parts[1] if len(parts) > 1 else "unavailable"


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def prefill_flops(net, P):
    from pytorchwavenetvocoder_b200.nets.wavenet import decode_prefill_windows
    R, ks, Ap = net.n_resch, net.kernel_size, net.n_aux_pad
    K1 = ks * R + Ap
    win = [min(s, P - 1) for s in decode_prefill_windows(net.dilations, ks)]
    return 2 * sum(win[l + 1] * (K1 * 2 * R + R * R) for l in range(len(win) - 1))


class Warmup(object):
    """The inputs and buffers of one streaming-decoder warm-up of B rows and seed length T0."""

    def __init__(self, net, B, T0):
        from pytorchwavenetvocoder_b200 import _lib
        from pytorchwavenetvocoder_b200.nets.wavenet import _decode_snapshot
        self.lib, self.net, self.B = _lib.load(), net, B
        self.P = max(T0, net.receptive_field)
        self.n_pad = self.P - T0
        U = net.upsampling_factor
        self.w, self.upw, self.upb = _decode_snapshot(net)
        self.wstream = net._decode_stream_pack(self.w)
        self.L = len(net.dilations)
        self.dil = (ctypes.c_int32 * self.L)(*net.dilations)
        g = torch.Generator(device="cuda").manual_seed(B)
        self.xs = torch.randint(0, 256, (B, self.P + 1), dtype=torch.int32, device="cuda", generator=g)
        self.h = torch.randn(B, net.n_aux, (self.P + U - 1) // U + 2, device="cuda", generator=g)
        self.queues = torch.zeros(self.lib.wnb_decode_workspace(B, net.n_resch, net.kernel_size, self.dil, self.L) // 4,
                                  device="cuda")
        self.nsm = torch.ones(B, dtype=torch.int32, device="cuda")

    def prefill(self):
        from pytorchwavenetvocoder_b200.nets.wavenet import _stream_prefill
        n = self.net
        _stream_prefill(self.lib, self.xs, self.P, self.h, self.upw, self.upb, self.w, self.wstream, self.dil, self.L,
                        self.queues, self.n_pad, n.n_quantize, n.n_aux, n.n_aux_pad, n.n_resch, n.n_skipch,
                        n.kernel_size, n.upsampling_factor)

    def sequential(self):
        from pytorchwavenetvocoder_b200 import _lib
        from pytorchwavenetvocoder_b200.nets.wavenet import MODE_SAMPLING, ptr, stream
        n, w = self.net, self.w
        _lib.check(self.lib.wnb_decode_stream_at(
            ptr(self.xs), ptr(self.h), ptr(self.upw), ptr(self.upb), ptr(w["wf"]), ptr(w["bf"]), ptr(self.wstream),
            ptr(w["b1"]), ptr(w["b2"]), ptr(w["bp1"]), ptr(w["bp2"]), self.dil, self.L, ptr(self.queues), ptr(self.nsm),
            None, None, self.B, self.P, 1, self.n_pad, self.h.size(2), n.n_quantize, n.n_aux, n.n_aux_pad, n.n_resch,
            n.n_skipch, n.kernel_size, n.upsampling_factor, MODE_SAMPLING, ctypes.c_uint64(1), 0, 0, 0, stream()),
            "decode_stream_at")


def model(cfg):
    from pytorchwavenetvocoder_b200.nets import WaveNet
    torch.manual_seed(0)
    net = WaveNet(*cfg).cuda().eval()
    assert net.decode_math == "fp32"
    return net


def part_a(out, sequential):
    for name, (cfg, fs) in SHAPES.items():
        net = model(cfg)
        for T0, prompt in ((1, "1 sample"), (5 * fs, "5 s")):
            for B in (1, 8, 64):
                wu = Warmup(net, B, T0)
                wu.prefill()
                t_pf = min(timed(wu.prefill) for _ in range(3))
                fl = prefill_flops(net, wu.P) * B
                row = dict(shape=name, prompt=prompt, B=B, P=wu.P, prefill_ms=t_pf * 1e3, prefill_gflop=fl / 1e9,
                           prefill_tflops=fl / t_pf / 1e12)
                if sequential and T0 == 1:
                    row["sequential_ms"] = timed(wu.sequential) * 1e3   # one run: it is slow
                    row["speedup"] = row["sequential_ms"] / row["prefill_ms"]
                print(json.dumps(row), flush=True)
                out.append(row)
                del wu
                torch.cuda.empty_cache()


def part_b(out):
    for name, (cfg, fs) in SHAPES.items():
        net = model(cfg)
        U = net.upsampling_factor
        h = torch.randn(1, net.n_aux, 2, device="cuda")
        x = torch.zeros(1, 1, dtype=torch.int64, device="cuda")

        def first():
            with torch.no_grad():
                s = net.decode_session(x, [10 * U], "sampling", seed=3)
                s.step(h).cpu()
        first()
        t = min(timed(first) for _ in range(3))
        row = dict(part="first_audio", shape=name, B=1, first_step_ms=t * 1e3)
        print(json.dumps(row), flush=True)
        out.append(row)


def part_cd(out):
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    net = model(SHAPES["arctic"][0])
    U, B, steps = net.upsampling_factor, 64, 480
    nf = 2 + (10 * steps) // U
    h = torch.randn(B, net.n_aux, nf, device="cuda")
    x = torch.zeros(B, 1, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        pool = net.decode_pool(B, "sampling", 5, kernel="stream")
        for k in range(B):
            pool.admit(x[k], 100 * steps, h[k], stream=k)
        pool.step(1)                            # admission
        pool.step(steps)                        # untimed call of the same shape
        t_pool = min(timed(lambda: pool.step(steps)) for _ in range(3))
        s = DecodeSession(net, x, [100 * steps] * B, "sampling", 5, None, False, "stream")
        s.step(h[:, :, :2])                     # warm-up and the first samples
        f0 = [2]

        def sess():
            s.step(h[:, :, f0[0]:f0[0] + steps // U])
            f0[0] += steps // U
        sess()
        t_sess = min(timed(sess) for _ in range(3))
    row = dict(part="pool_vs_session", shape="arctic", B=B, steps=steps, pool_call_ms=t_pool * 1e3,
               session_step_ms=t_sess * 1e3, pool_ms_per_step=t_pool * 1e3 / steps, session_ms_per_step=t_sess * 1e3 / steps)
    print(json.dumps(row), flush=True)
    out.append(row)
    with torch.no_grad():
        for k_admit in (1, 8, 64):
            pool = net.decode_pool(B, "sampling", 5, kernel="stream")
            for k in range(B - k_admit):
                pool.admit(x[k], 100 * steps, h[k], stream=k)
            pool.step(1)
            pool.step(1)
            t_steady = min(timed(lambda: pool.step(1)) for _ in range(3))
            times = []
            for rep in range(3):
                for k in range(k_admit):
                    pool.admit(x[0], 10, h[0], stream=1000 * (rep + 1) + k)
                times.append(timed(lambda: pool.step(1)))
                while any(not pool.finished(1000 * (rep + 1) + k) for k in range(k_admit)):
                    pool.step(16)
            row = dict(part="admission", shape="arctic", capacity=B, admitted=k_admit, admit_call_ms=min(times) * 1e3,
                       steady_1step_call_ms=t_steady * 1e3)
            print(json.dumps(row), flush=True)
            out.append(row)


def part_e(out):
    """The prefill against the sequential warm-up at short warm-ups: both followed by nothing (the sequential one
    includes one decoded step, as in part a)."""
    for cfg in ((256, 28, 64, 512, 4, 2, 2, 4), (256, 28, 64, 64, 4, 2, 3, 4), (256, 28, 512, 256, 4, 1, 2, 80)):
        net = model(cfg)
        rf = net.receptive_field
        for T0 in sorted({1, 64, 128, 256, 512, 1024, 2 * rf}):
            for B in (1, 5, 64):
                wu = Warmup(net, B, T0)
                wu.prefill()
                wu.sequential()
                t_pf = sorted(timed(wu.prefill) for _ in range(5))[2]
                t_sq = sorted(timed(wu.sequential) for _ in range(5))[2]
                row = dict(part="short_warmup", cfg=list(cfg), rf=rf, B=B, warmup_positions=wu.P - 1,
                           prefill_ms=t_pf * 1e3, sequential_ms=t_sq * 1e3)
                print(json.dumps(row), flush=True)
                out.append(row)
                del wu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--no-sequential", action="store_true")
    ap.add_argument("--parts", default="abcd")
    args = ap.parse_args()
    name, power, clock = card()
    print(json.dumps(dict(card=name, power_limit=power, sm_clock=clock)), flush=True)
    out = [dict(card=name, power_limit=power, sm_clock=clock)]
    if "a" in args.parts:
        part_a(out, not args.no_sequential)
    if "b" in args.parts:
        part_b(out)
    if "c" in args.parts or "d" in args.parts:
        part_cd(out)
    if "e" in args.parts:
        part_e(out)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
