#!/usr/bin/env python
# -*- coding: utf-8 -*-
"""bench.py -- the benchmark of the WaveNet hot paths on the H100.

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload train|decode] [--dump-outputs DIR]

Default workload = BASELINE.json configs[1]: arctic/sd 16 kHz, 3x10 dilation layers, 64 res / 512 skip,
mu-law 256, aux 28 + UpSampling(80), batch 8 x 23 040-sample windows (20 000 nominal + receptive field,
reference bin/train.py:106-110) per GPU.  One "step" = forward + cross-entropy + backward + Adam step of
that batch (reference bin/train.py:530-540) through ``pytorchwavenetvocoder_b200.nets.WaveNet``.

  value   = train waveform-samples/s with the batch resident in HBM (whole job, all ranks);
  e2e     = the same step fed from pinned HOST buffers (H2D of x,h,t inside the timed region) and with
            the loss read back to the host every step (the call a user of bin/train.py makes);
  decode  = (extra object) persistent fast-generate kernel, configs[3] shape (64 utterances), bounded
            number of samples per utterance -- stated in the object;
  roofline= fused residual-block FORWARD kernel: algorithmic bytes s*(2R + A + 2S) per sample-layer
            (SURVEY.md 8d; 4 720 B fp32 at 64/512/28) x B*T per launch / mean launch time (CUDA events on
            the launching stream, inside the timed steps) against MEASURED_PEAKS.json hbm_gbs (else the H100 SXM
            data-sheet 3.35 TB/s, reported as "fallback");
  cpu_baseline / --impl reference = oracle/torch_port.py (the reference's op sequence on torch CPU, all
            host threads) on a bounded sample (1 window per step).

--dump-outputs DIR writes, after the timed steps, what the last timed step computed as DIR/<name>.npy (float32 /
float64, <= 64 MB in all): the loss, every parameter after the optimizer step and its gradient, and with the decode
workload the generated samples.  Inputs and weights are seeded, so two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CFG = (256, 28, 64, 512, 10, 3, 2, 80)       # BASELINE.json configs[1] / north_star shape
BATCH, BATCH_LENGTH = 8, 20000
FALLBACK_HBM_GBS = 3350.0      # H100 SXM data sheet (HBM3); MEASURED_PEAKS.json overrides


def _peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "measured"
    except Exception:
        return FALLBACK_HBM_GBS, "fallback"


def _tensor_peak():
    """Sustained dense bf16 TFLOP/s of MEASURED_PEAKS.json (cuBLAS, back to back); tf32 runs at half that rate."""
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["bf16_tflops_sustained"]), "measured"
    except Exception:
        return 989.0, "fallback"      # H100 SXM data sheet, dense BF16


class ClockSampler(object):
    """nvidia-smi clocks/throttle reasons sampled DURING the timed region."""

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if len(r) >= 6 and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) >= 6 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) >= 6 and r[2 + i].lower().startswith("active")
                                                         for r in self.rows)]
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


class _Cfg(object):
    """Plain view of the WaveNet ctor tuple (no oracle import on the measured arm)."""

    def __init__(self, t):
        (self.n_quantize, self.n_aux, self.n_resch, self.n_skipch, self.dilation_depth, self.dilation_repeat,
         self.kernel_size, self.upsampling_factor) = t
        self.dilations = [2 ** i for i in range(self.dilation_depth)] * self.dilation_repeat
        self.receptive_field = (self.kernel_size - 1) * sum(self.dilations) + 1


def make_model(device, math_mode, seed=20260924):
    """Random-init weights of the named architecture: the reference initialiser (xavier conv weights, unit
    up-sampling) plus seeded N(0, 0.05) biases so that no bias path is trivially zero (SURVEY.md 8d)."""
    from pytorchwavenetvocoder_b200.nets import WaveNet, initialize
    cfg = _Cfg(CFG)
    torch.manual_seed(seed)
    net = WaveNet(*CFG)
    net.apply(initialize)
    with torch.no_grad():
        for name, prm in net.named_parameters():
            if name.endswith("bias"):
                prm.add_(0.05 * torch.randn_like(prm))
    net.math_mode = math_mode
    return cfg, net.to(device)


def synth_batch(cfg, rank, B, pinned):
    g = torch.Generator().manual_seed(20260924 + rank)
    T = BATCH_LENGTH + cfg.receptive_field - 1 + 1          # bin/train.py:106-110 -> 23 069 -> trimmed below
    T = (T // cfg.upsampling_factor) * cfg.upsampling_factor  # validate_length: multiple of U -> 23 040
    xfull = torch.randint(0, cfg.n_quantize, (B, T + 1), generator=g, dtype=torch.int64)
    x, t = xfull[:, :-1].contiguous(), xfull[:, 1:].contiguous()
    h = torch.randn(B, cfg.n_aux, T // cfg.upsampling_factor, generator=g)
    if pinned:
        x, t, h = x.pin_memory(), t.pin_memory(), h.pin_memory()
    return x, h, t


def run_ours(args):
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        # NCCL prints its version banner on stdout while the communicator is created: send fd 1 to stderr for
        # that moment so that stdout carries nothing but the one JSON line
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(2, 1)
        try:
            dist.init_process_group("nccl", device_id=dev)
            dist.barrier()
            torch.cuda.synchronize()
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    from pytorchwavenetvocoder_b200.nets import wavenet as wn
    _lib.load()

    out = {}
    if args.workload == "train":
        cfg, net = make_model(dev, args.math)
        net.train()
        if world > 1:
            from pytorchwavenetvocoder_b200.parallel import GradAllReduce
            sync = GradAllReduce(net)
        else:
            sync = None
        # torch.optim.Adam (reference bin/train.py:457-460) whose step is one wnb_adam_flat launch over the flat gradient
        # buffer; WNB_TORCH_ADAM=1: torch's own fused multi-tensor step (A/B runs)
        if os.environ.get("WNB_TORCH_ADAM") == "1":
            opt = torch.optim.Adam(net.parameters(), lr=1e-4, fused=True)
        else:
            from pytorchwavenetvocoder_b200.optim import Adam as WnbAdam
            opt = WnbAdam(net.parameters(), lr=1e-4, module=net)
        xh, hh, th = synth_batch(cfg, rank, BATCH, pinned=True)
        xd, hd, td = xh.to(dev), hh.to(dev), th.to(dev)
        rf = cfg.receptive_field

        def step(x, h, t):
            loss = net.forward_loss(x, h, t, rf)     # = cross_entropy(net(x, h), t, rf) as one autograd node
            opt.zero_grad(set_to_none=True)
            loss.backward()
            if sync is not None:
                sync.allreduce()
            opt.step()
            return loss

        def barrier():
            torch.cuda.synchronize()
            if dist is not None:
                dist.barrier()
                torch.cuda.synchronize()

        sampler = ClockSampler(local)     # samples clocks under load: warm-up + timed region
        if rank == 0:
            sampler.start()
        for _ in range(args.warmup):
            step(xd, hd, td)
        # --- device-resident timing (value) ---
        barrier()
        l0 = _lib.launch_count()
        lib = _lib.load()
        L = len(net.dilations)
        stack = bool(args.math == "tf32" and lib.wnb_stack_supported(cfg.n_resch, cfg.n_skipch, net.n_aux_pad,
                                                                     cfg.kernel_size, L, _lib.MATH_TF32))
        if not stack:
            wn.PROFILE_EVENTS = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            loss = step(xd, hd, td)
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        launches = _lib.launch_count() - l0
        if args.dump_outputs and rank == 0:     # (outside the timed region; the steps after this one do not change it)
            DUMP["loss"] = loss.detach().double().cpu().numpy().reshape(1)
            for name, prm in net.named_parameters():
                DUMP["param." + name] = prm.detach().float().cpu().numpy()
                if prm.grad is not None:
                    DUMP["grad." + name] = prm.grad.detach().float().cpu().numpy()
        evs = wn.PROFILE_EVENTS or []
        wn.PROFILE_EVENTS = None
        blk_ms = [a.elapsed_time(b) for a, b in evs]
        kinds = []
        if stack:
            # Per-kernel durations for the roofline block: the product path is ONE ABI call per direction
            # (csrc/stack.cu), which brackets each of its launches with CUDA events on the launching stream while
            # wnb_profile_enable(1) is on.  Those event records sit between the kernels, cost ~3 % and defeat the
            # programmatic-dependent-launch overlap, so they run on `steps` EXTRA steps right after the timed region
            # (same buffers, same clocks) instead of inside it.
            import ctypes
            _lib.check(lib.wnb_profile_enable(1), "profile_enable")
            ep0, ep1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ep0.record()
            for _ in range(args.steps):
                step(xd, hd, td)
            ep1.record()
            barrier()
            ms_prof = ep0.elapsed_time(ep1)
            for k, name in enumerate(STACK_KINDS):
                tot, n = ctypes.c_double(0.0), ctypes.c_int(0)
                _lib.check(lib.wnb_profile_read(k, ctypes.byref(tot), ctypes.byref(n)), "profile_read")
                kinds.append((name, tot.value, n.value))
            _lib.check(lib.wnb_profile_enable(0), "profile_enable")
        clocks = sampler.stop() if rank == 0 else None
        # --- end-to-end timing: pinned host -> device every step, loss read back every step ---
        # The public-API loop a trainer runs (bin/train.py): the next batch's host->device copy is issued on a copy
        # stream before the current loss is read back (what the reference's background batch generator does with
        # its prefetch thread), so each step's copy overlaps the previous step's kernels; every step still copies its
        # own inputs from pinned memory and reads its own loss inside the timed region.
        copy_stream = torch.cuda.Stream(device=dev)

        def fetch():
            with torch.cuda.stream(copy_stream):
                tens = (xh.to(dev, non_blocking=True), hh.to(dev, non_blocking=True), th.to(dev, non_blocking=True))
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            return tens, ev

        def e2e_loop(n):
            # every step's loss is read back to the host inside the loop, one step late (the usual logging lag of a
            # training loop: the host stays one step ahead of the device instead of draining it every iteration)
            last_loss, pending = 0.0, None
            nxt = fetch()
            for i in range(n):
                (xb, hb, tb), ev = nxt
                cur = torch.cuda.current_stream()
                cur.wait_event(ev)
                for tns in (xb, hb, tb):
                    tns.record_stream(cur)
                loss_i = step(xb, hb, tb)
                if i + 1 < n:
                    nxt = fetch()
                if pending is not None:
                    last_loss = float(pending)
                pending = loss_i.detach()
            return float(pending)

        e2e_loop(2)
        barrier()
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        last = e2e_loop(args.steps)
        e3.record()
        barrier()
        ms_e2e = e2.elapsed_time(e3)
        # --- end-to-end through the CLI's data path (bin/train.py): DISTINCT batches every step from wav / feature
        # FILES -> reader thread -> pinned memory -> async H2D into the device rings -> wnb_make_train_batch
        # (windowing + mu-law + scaler on the device) -> step; loss read back one step late as above ---
        loader_e2e = None
        if args.loader_e2e and cfg.upsampling_factor > 0:
            import shutil
            import tempfile
            from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav
            from pytorchwavenetvocoder_b200.utils.device_loader import DeviceTrainGenerator
            tmpd = tempfile.mkdtemp(prefix="wnb_bench_")
            try:
                rngc = np.random.RandomState(1000 + rank)
                U, n_utt, n_frames = cfg.upsampling_factor, 24, 2000      # 24 utterances x 10 s @ 16 kHz
                wl, fl = [], []
                for i in range(n_utt):
                    w, f = os.path.join(tmpd, "u%d.wav" % i), os.path.join(tmpd, "u%d.npz" % i)
                    write_wav(w, 0.5 * np.tanh(rngc.standard_normal(n_frames * U)), 16000)
                    write_hdf5(f, "/world", rngc.standard_normal((n_frames, cfg.n_aux)).astype(np.float32))
                    wl.append(w)
                    fl.append(f)
                gen = DeviceTrainGenerator(wl, fl, rf, BATCH_LENGTH, BATCH, n_quantize=cfg.n_quantize,
                                           mean=np.zeros(cfg.n_aux), scale=np.ones(cfg.n_aux), shuffle=True,
                                           upsampling_factor=U, use_upsampling_layer=True, device=local)

                def loader_loop(n):
                    pending, last_ = None, 0.0
                    for _ in range(n):
                        (xb, hb), tb = gen.next()
                        loss_i = step(xb, hb, tb)
                        if pending is not None:
                            last_ = float(pending)
                        pending = loss_i.detach()
                    return float(pending)
                loader_loop(3)
                barrier()
                gen.stats.update(reader_s=0.0, utts=0, wait_s=0.0, batches=0, launch_s=0.0)   # steady state only
                e4, e5 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s0_ = gen.tail_s
                e4.record()
                last_l = loader_loop(args.steps)
                e5.record()
                barrier()
                ms_l = e4.elapsed_time(e5)
                up_bytes = (gen.tail_s - s0_) * (4 + cfg.n_aux * 4.0 / U)
                loader_e2e = {"ms": ms_l, "last_loss": last_l, "h2d_bytes_per_step": int(up_bytes / args.steps),
                              "T": gen.T, "reader_ms_per_utterance": 1e3 * gen.stats["reader_s"] / max(gen.stats["utts"], 1),
                              "consumer_wait_ms_per_batch": 1e3 * gen.stats["wait_s"] / max(gen.stats["batches"], 1),
                              "launch_ms_per_batch": 1e3 * gen.stats.get("launch_s", 0.0) / max(gen.stats["batches"], 1),
                              "reader_threads": gen.n_readers}
            finally:
                shutil.rmtree(tmpd, ignore_errors=True)
        fp32_line = None
        if args.fp32_line and args.math == "tf32" and world == 1:
            # the parity mode beside the tensor-core number: same model, same batch, math_mode = "fp32" (FFMA kernels,
            # logits <= 1e-4 / gradients <= 1e-3 vs the reference), 1 warm-up + 2 timed steps
            net.math_mode = "fp32"
            step(xd, hd, td)
            barrier()
            ef0, ef1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ef0.record()
            for _ in range(2):
                step(xd, hd, td)
            ef1.record()
            barrier()
            net.math_mode = args.math
            msf = ef0.elapsed_time(ef1) / 2
            fp32_line = {"ms_per_step": msf, "value": BATCH * BATCH_LENGTH / (msf * 1e-3), "unit": "samples/s",
                         "dtype": "f32", "steps": 2,
                         "note": "math_mode=fp32: every contraction in fp32 FFMA (the parity path of the tests)"}
        if dist is not None:
            tt = torch.tensor([ms, ms_e2e, loader_e2e["ms"] if loader_e2e else 0.0], device=dev, dtype=torch.float64)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            ms, ms_e2e = float(tt[0]), float(tt[1])
            if loader_e2e:
                loader_e2e["ms"] = float(tt[2])
        per_step = ms / args.steps
        samples = world * BATCH * BATCH_LENGTH
        hbm, how = _peaks()
        Bq, T = xd.shape
        s, R, S, A = 4, cfg.n_resch, cfg.n_skipch, cfg.n_aux
        alg_bytes = float(Bq) * T * s * (2 * R + A + 2 * S)
        blk = float(np.mean(blk_ms)) if blk_ms else None
        ach = alg_bytes / (blk * 1e-3) / 1e9 if blk else None
        roof = {"kernel": "resblock_fwd (%s)" % args.math, "bound": "hbm", "achieved": ach, "peak": hbm,
                "unit": "GB/s", "frac": (ach / hbm) if ach else None, "traffic": None,
                "peak_source": how, "algorithmic_bytes_per_launch": alg_bytes,
                "mean_launch_ms": blk, "launches_timed": len(blk_ms)}
        if not stack and args.math == "tf32" and R * R >= 256 * 256:
            # shapes of the composed path (the recipes' 512 res / 256 skip): tensor-bound (AI 470 flop/B, SURVEY 8d) -- the
            # whole step's GEMM FLOPs against the tf32 rate (half the measured sustained bf16 rate)
            ks_, Q_ = cfg.kernel_size, cfg.n_quantize
            fwd = L * (2.0 * R * R * (2 * ks_ + 1) + 4.0 * R * A + 2.0 * S * R) + 2.0 * S * S + 2.0 * Q_ * S
            flops = 3.0 * fwd * float(Bq) * T
            pk, pk_how = _tensor_peak()
            ach_tf = flops / (per_step * 1e-3) / 1e12
            roof = {"kernel": "whole step: every GEMM of the composed tensor-core path (gemm_nt_tc / wgrad_tc kernels)",
                    "bound": "tensor", "achieved": ach_tf, "peak": pk / 2, "unit": "TFLOP/s", "frac": ach_tf / (pk / 2),
                    "traffic": None, "peak_source": pk_how + " bf16_tflops_sustained / 2 (tf32 rate)",
                    "flops_per_step": flops,
                    "note": "fwd FLOPs/sample = L*[2R^2(2ks+1)+4RA+2SR]+2S^2+2QS (SURVEY 8d), backward = 2x"}
        roof_all = None
        if stack:
            # algorithmic bytes per launch of every kernel kind of the deferred-skip stack (DESIGN.md section 4):
            # fp32 channels-last tensors, each streamed once; weights (<= 4 MB) not counted
            bt4, Ap, LR = float(Bq) * T * 4, net.n_aux_pad, L * R
            alg = {"fwd_block": bt4 * (3 * R + Ap), "skip_gemm": bt4 * (LR + S), "dzall_gemm": bt4 * (S + LR),
                   "gate_bwd": bt4 * (5 * R + Ap), "dx_gemm": bt4 * (4 * R + 2 * Ap),
                   # every block's dW1 / dW2res in ONE segmented launch each (dpre_l, x_l, aux | dout_l, z_l)
                   # (aux is shared by all blocks and stays in L2: counted once)
                   "dw1": L * bt4 * 3 * R + bt4 * Ap, "dw2res": (L - 1) * bt4 * 2 * R, "dwskip": bt4 * (S + LR)}
            roof_all = []
            for name, tot, n in kinds:
                if n == 0:
                    continue
                mean = tot / n
                a = alg[name] / (mean * 1e-3) / 1e9
                roof_all.append({"kernel": name, "launches_timed": n, "mean_launch_ms": mean,
                                 "share_of_step": tot / ms_prof, "algorithmic_bytes_per_launch": alg[name],
                                 "achieved": a, "frac": a / hbm, "traffic": None})
            # the four per-block backward kernels against what ONE fused kernel per block would have to move
            # (x, dout, dZ_all slice, aux in; dx out = s*(4R+Ap) per sample; DESIGN.md 3.1 says why it is not built)
            byk = {r["kernel"]: r for r in roof_all}
            fused_ideal = None
            if all(k in byk for k in ("gate_bwd", "dx_gemm", "dw1", "dw2res")):
                t_blk = (byk["gate_bwd"]["mean_launch_ms"] + byk["dx_gemm"]["mean_launch_ms"]
                         + byk["dw1"]["mean_launch_ms"] / L + byk["dw2res"]["mean_launch_ms"] / max(L - 1, 1))
                ideal = bt4 * (4 * R + Ap)
                fused_ideal = {"bytes_per_block": ideal, "ms_per_block_now": t_blk,
                               "achieved": ideal / (t_blk * 1e-3) / 1e9, "frac": ideal / (t_blk * 1e-3) / 1e9 / hbm,
                               "note": "gate_bwd + dx + dW1/L + dW2res/(L-1) per block vs s*(4R+Ap)*B*T"}
            top = max(roof_all, key=lambda r: r["share_of_step"])
            roof = {"kernel": "%s (tf32, deferred-skip stack)" % top["kernel"], "bound": "hbm", "achieved": top["achieved"],
                    "peak": hbm, "unit": "GB/s", "frac": top["frac"], "traffic": top["traffic"], "peak_source": how,
                    "algorithmic_bytes_per_launch": top["algorithmic_bytes_per_launch"],
                    "mean_launch_ms": top["mean_launch_ms"], "launches_timed": top["launches_timed"],
                    "share_of_step": top["share_of_step"], "fused_ideal": fused_ideal,
                    "measured_on": "%d extra steps after the timed region with per-launch CUDA events "
                                   "(%.3f ms/step there; the events stay out of the timed steps)"
                                   % (args.steps, ms_prof / args.steps)}
        out = {
            "metric": "train waveform-samples/s (fwd+CE+bwd+Adam), arctic/sd 30-layer 64res/512skip",
            "value": samples / (per_step * 1e-3), "unit": "samples/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": per_step, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "tf32" if args.math == "tf32" else "f32", "data": "synthetic",
            "config": {"workload": ("configs[1]: arctic/sd 16kHz " if CFG == (256, 28, 64, 512, 10, 3, 2, 80) else "custom: ") +
                                   "WaveNet%s batch %d x %d (nominal batch length + rf window) per GPU, Adam, loss on [rf:]"
                                   % (str(CFG).replace(" ", ""), BATCH, int(T)),
                       "global_batch": world * BATCH, "seq_len": int(T), "parallelism": "dp%d" % world,
                       "math": args.math, "storage": "fp32 channels-last",
                       "l2": "per-step working set ~10 GB >> 50 MB L2 (no explicit flush needed)"},
            "e2e": {"value": samples / (ms_e2e / args.steps * 1e-3), "unit": "samples/s",
                    "h2d_bytes_per_step": int(xh.numel() * 8 + th.numel() * 8 + hh.numel() * 4),
                    "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps, "last_loss": last,
                    "loop": "next batch copied H2D on a copy stream while the step runs; each step's loss read back "
                            "one step later (all %d reads inside the timed region)" % args.steps},
            "gpu_launches": int(launches),
            "clocks": clocks,
            "roofline": roof,
        }
        if fp32_line:
            out["fp32_parity_mode"] = fp32_line
        if loader_e2e:
            out["e2e_data_loader"] = {
                "value": samples / (loader_e2e["ms"] / args.steps * 1e-3), "unit": "samples/s",
                "ms_per_step": loader_e2e["ms"] / args.steps, "h2d_bytes_per_step": loader_e2e["h2d_bytes_per_step"],
                "d2h_bytes_per_step": 4, "last_loss": loader_e2e["last_loss"],
                "reader_ms_per_utterance": loader_e2e["reader_ms_per_utterance"],
                "consumer_wait_ms_per_batch": loader_e2e["consumer_wait_ms_per_batch"],
                "launch_ms_per_batch": loader_e2e["launch_ms_per_batch"],
                "reader_threads": loader_e2e["reader_threads"],
                "loop": "bin/train.py's data path: distinct batches every step cut on the device "
                        "(wnb_make_train_batch) from 24 synthetic 10 s wav + feature files read by the loader thread, "
                        "uploaded once per utterance from pinned memory on a copy stream; window %d samples"
                        % loader_e2e["T"]}
        if roof_all:
            out["roofline_kernels"] = roof_all
    if args.workload == "decode" or (args.workload == "train" and args.with_decode):
        dec = run_decode(args, dev, rank, world, dist)
        if args.workload == "decode":
            out = dec
        else:
            out["decode"] = dec
    if rank == 0:
        if args.dump_outputs:
            write_dump(args.dump_outputs)
        if world == 1 and args.cpu_baseline:
            out["cpu_baseline"] = cpu_baseline(args, out.get("config", {}).get("workload", ""),
                                               decode=(args.workload == "decode"))
        print(json.dumps(out))
    if dist is not None:
        dist.destroy_process_group()


# kernel kinds timed by wnb_profile_read (WNB_PROF_* order)
STACK_KINDS = ["fwd_block", "skip_gemm", "dzall_gemm", "gate_bwd", "dx_gemm", "dw1", "dw2res", "dwskip"]


DUMP = {}                       # name -> array: what the last timed step computed (--dump-outputs)
DUMP_BUDGET = 63 * 1024 * 1024       # (+ the .npy headers: <= 64 MB in all)


def write_dump(out_dir):
    """DUMP -> out_dir/<name>.npy.  If the arrays exceed DUMP_BUDGET in all, the largest ones are replaced by a fixed,
    seeded sample of their elements (<name>.npy, flattened) with the sampled flat indices in <name>.index.npy."""
    os.makedirs(out_dir, exist_ok=True)
    arrays = dict(DUMP)
    total = sum(a.nbytes for a in arrays.values())
    for name in sorted(arrays, key=lambda k: -arrays[k].nbytes):
        if total <= DUMP_BUDGET:
            break
        a = arrays[name]
        keep = (DUMP_BUDGET - (total - a.nbytes)) // (a.itemsize + 8)      # sampled values + float64 indices
        keep = min(a.size, keep if keep > 0 else 1 << 16)                   # (<= 0: the next arrays are sampled too)
        idx = np.sort(np.random.RandomState(0).choice(a.size, size=keep, replace=False))
        arrays[name] = a.reshape(-1)[idx]
        arrays[name + ".index"] = idx.astype(np.float64)
        total = sum(v.nbytes for v in arrays.values())
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def run_decode(args, dev, rank, world, dist):
    """configs[3]/[4]: batch autoregressive decode, utterances sharded over ranks (reference decode.py:261)."""
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = make_model(dev, "fp32")
    net.eval()
    n_utt_total = args.decode_utts * world        # weak scaling: fixed utterances per GPU
    n = args.decode_samples
    g = torch.Generator().manual_seed(20260924 + rank)
    U = cfg.upsampling_factor
    frames = (n + 1 + U - 1) // U
    h_host = torch.randn(args.decode_utts, cfg.n_aux, frames, generator=g).pin_memory()
    x_host = torch.full((args.decode_utts, 1), cfg.n_quantize // 2, dtype=torch.int64).pin_memory()
    nl = [n] * args.decode_utts

    def once(host, n_run=None):
        nlr = nl if n_run is None else [n_run] * args.decode_utts
        if host:
            x, h = x_host.to(dev, non_blocking=True), h_host.to(dev, non_blocking=True)
        else:
            x, h = once.xd, once.hd
        gen = net._decode(x, h, nlr, "sampling", seed=1234)
        if host:
            return gen.cpu()
        return gen
    once.xd, once.hd = x_host.to(dev), h_host.to(dev)
    lib = _lib.load()
    with torch.no_grad():
        once(False, min(n, 2000))      # warm-up: a short run of the same kernel (one-time initialisation, clocks)
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        l0 = _lib.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gen_timed = once(False)
        e1.record()
        torch.cuda.synchronize()
        launches = _lib.launch_count() - l0
        if args.dump_outputs and rank == 0:
            DUMP["decode.samples"] = gen_timed.float().cpu().numpy()   # mu-law codes < 2^24: exact in float32
        ms = e0.elapsed_time(e1)
        t0 = time.time()
        once(True)
        torch.cuda.synchronize()
        ms_e2e = (time.time() - t0) * 1e3
    if dist is not None:
        tt = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        ms, ms_e2e = float(tt[0]), float(tt[1])
    steps_incl_warmup = n + cfg.receptive_field - 1
    wbytes = sum(p.numel() for p in net.parameters()) * 4
    kern = getattr(net, "last_decode_kernel", None)
    cl = int(lib.wnb_decode_warp_cluster(args.decode_utts)) if kern == "warp" else 1
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    nu = 1 if args.decode_utts <= sms else (2 if args.decode_utts <= 2 * sms else 4)
    ctas = (args.decode_utts + nu - 1) // nu * cl
    us_step = ms * 1e3 / steps_incl_warmup
    sm_mhz = 1980.0      # H100 SXM boost clock; MEASURED_PEAKS.json sm_max_mhz overrides
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            sm_mhz = float(json.load(f).get("sm_max_mhz", sm_mhz))
    except Exception:
        pass
    cyc_step = us_step * sm_mhz
    # the recurrence is a per-sample dependency chain, not an HBM stream (SURVEY.md 8d "roofline -- decode"): what bounds a
    # step is how fast ONE SM can pull its share of the 8.6 MB of weights through L2 -> shared memory and read it once
    # with the FFMA GEMVs (128 B/clk shared-memory pipe); the HBM traffic per generated sample is < 10 B
    per_cta_bytes = wbytes / cl
    roof = {"bound": "per-sample dependency chain; per-SM L2->smem weight stream",
            "kernel": "decode_%s_kernel, %d CTA(s) per utterance, %d CTAs on %d SMs" % (kern, cl, ctas, sms),
            "us_per_step": us_step, "sm_cycles_per_step": cyc_step,
            "smem_read_floor_cycles": per_cta_bytes / 128.0,
            "frac_of_smem_floor": (per_cta_bytes / 128.0) / cyc_step,
            "weight_stream_bytes_per_clk_per_sm": per_cta_bytes / cyc_step,
            "l2_to_sm_weight_stream_GBps": ctas * per_cta_bytes / (us_step * 1e-6) / 1e9,
            "algorithmic_hbm_bytes_per_sample": 4.0 * cfg.n_aux / max(U, 1) + 8.0,
            "flops_per_sample": 4.2e6, "achieved_tflops": n_utt_total * n / (ms * 1e-3) * 4.2e6 / 1e12,
            "dram_bytes_ncu": None}
    return {
        "metric": "autoregressive decode samples/s (persistent fast-generate kernel, sampling mode)",
        "value": n_utt_total * n / (ms * 1e-3), "unit": "samples/s", "n_gpus": world,
        "ms": ms, "higher_is_better": True, "scaling": "weak", "dtype": "f32", "data": "synthetic",
        "config": {"workload": "configs[3]: %d utterances/GPU x %d samples%s, arctic/sd "
                               "30-layer 64/512, seed 128, aux N(0,1)"
                               % (args.decode_utts, n, "" if n >= 159999 else " (bounded from 159999)"),
                   "utterances": n_utt_total, "samples_per_utterance": n,
                   "warmup_steps_in_time": cfg.receptive_field - 1},
        "us_per_step": us_step,
        "weight_stream_GBps": (args.decode_utts * steps_incl_warmup * wbytes) / (ms * 1e-3) / 1e9,
        "roofline": roof,
        "e2e": {"value": n_utt_total * n / (ms_e2e * 1e-3), "unit": "samples/s",
                "h2d_bytes_per_step": int(h_host.numel() * 4 + x_host.numel() * 8),
                "d2h_bytes_per_step": int(args.decode_utts * n * 4)},
        "gpu_launches": int(launches),
    }


def cpu_baseline(args, workload, decode=False, steps=None):
    """The reference's op sequence restated on torch CPU ops (oracle/torch_port.py, kind "port") on the host cores;
    bounded sample."""
    from oracle import torch_port as TP
    from oracle import wavenet_oracle as O
    cores = min(os.cpu_count() or 1, 16)
    torch.set_num_threads(cores)
    cfg = O.Config(*CFG)
    if decode:
        p = TP.params_to_torch(O.make_params(cfg, 20260924))
        B = 8
        g = torch.Generator().manual_seed(1)
        x = torch.full((B, 1), 128, dtype=torch.int64)

        def run(n):
            h = torch.randn(B, cfg.n_aux, (n + 1 + 79) // 80, generator=g)
            t0 = time.time()
            TP.batch_fast_generate(cfg, p, x, h, [n] * B, "argmax")
            return time.time() - t0
        a, b = run(20), run(60)
        v = B * 40 / max(b - a, 1e-9)
        return {"value": v, "unit": "samples/s", "cores": cores, "kind": "port",
                "sample": "batch_fast_generate B=8, 60 vs 20 samples differenced, torch CPU fp32"}
    p = TP.params_to_torch(O.make_params(cfg, 20260924), requires_grad=True)
    opt = torch.optim.Adam(list(p.values()), lr=1e-4)
    x, h, t = synth_batch(cfg, 0, 1, pinned=False)
    t0 = time.time()
    TP.train_step(cfg, p, opt, x, h, t)
    warm = time.time() - t0
    k = steps or 2
    if warm > 15.0 and steps is None:
        k, dt = 1, warm
    else:
        t0 = time.time()
        for _ in range(k):
            TP.train_step(cfg, p, opt, x, h, t)
        dt = (time.time() - t0) / k
    return {"value": BATCH_LENGTH / dt, "unit": "samples/s", "cores": cores, "kind": "port",
            "sample": "%d step(s) of 1 x 23040-sample window (fwd+CE+bwd+Adam), torch CPU fp32, after 1 warm-up" % k,
            "sec_per_step": dt}


def run_reference(args):
    rank = int(os.environ.get("RANK", 0))
    if rank != 0:
        return
    cfg = _Cfg(CFG)
    decode = args.workload == "decode"
    k = max(1, args.steps)
    cb = cpu_baseline(args, "", decode=decode, steps=k)
    world = int(os.environ.get("WORLD_SIZE", 1))
    out = {
        "impl": "reference",
        "metric": ("autoregressive decode samples/s" if decode else
                   "train waveform-samples/s (fwd+CE+bwd+Adam), arctic/sd 30-layer 64res/512skip"),
        "value": cb["value"], "unit": "samples/s", "n_gpus": world, "steps": k, "warmup": 1,
        "ms_per_step": cb.get("sec_per_step", 0) * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "configs[1] arctic/sd WaveNet(256,28,64,512,10,3,2,80); bounded sample: " + cb["sample"],
                   "receptive_field": cfg.receptive_field},
        "cpu_baseline": cb,
        "e2e": {"value": cb["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5,
                    help="timed training steps (the decode leg always times one full decode of --decode-utts utterances)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="train", choices=["train", "decode"])
    ap.add_argument("--math", default=None, choices=["fp32", "tf32"])
    ap.add_argument("--with-decode", type=int, default=1, help="also report the decode workload (extra object)")
    ap.add_argument("--cpu-baseline", type=int, default=1)
    ap.add_argument("--loader-e2e", type=int, default=1, help="also time the step fed by the on-device data loader")
    ap.add_argument("--cfg", default=None, help="override the WaveNet ctor tuple, e.g. 256,28,512,256,10,3,2,80 "
                                                "(recipe shape); the default is BASELINE.json configs[1]")
    ap.add_argument("--batch", type=int, default=None, help="override the per-GPU batch (default 8)")
    ap.add_argument("--decode-utts", type=int, default=64)
    ap.add_argument("--decode-samples", type=int, default=159999,
                    help="samples per utterance (configs[3]: 2000 frames x 80 - 1 = 159 999, reference decode.py:158)")
    ap.add_argument("--batch-length", type=int, default=None, help="override the nominal batch length (default 20000)")
    ap.add_argument("--fp32-line", type=int, default=1, help="also time a few steps of the fp32 FFMA parity mode")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed to DIR/<name>.npy")
    args = ap.parse_args()
    global CFG, BATCH, BATCH_LENGTH
    if args.batch_length:
        BATCH_LENGTH = args.batch_length
    if args.cfg:
        CFG = tuple(int(v) for v in args.cfg.split(","))
    if args.batch:
        BATCH = args.batch
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        return run_reference(args)
    if args.math is None:
        from pytorchwavenetvocoder_b200.nets.wavenet import tc_supported
        args.math = "tf32" if tc_supported(CFG) else "fp32"
    run_ours(args)


if __name__ == "__main__":
    main()
