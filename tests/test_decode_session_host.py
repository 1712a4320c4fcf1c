# -*- coding: utf-8 -*-
"""CPU tier: resumable decoding without a GPU.

* ``nets.wavenet.decode_window`` (the host arithmetic every ``DecodeSession.step`` uses) drives the float FIFO oracle
  (``oracle.FifoState`` / ``fifo_step``) chunk by chunk, giving each call only what the window says it reads -- the xs
  columns from ``xs_base``, the aux frames from ``h_frame0``, the call's slice of the uniforms -- and must reproduce
  ``oracle.batch_fast_generate`` exactly: kernel sizes 2 and 3, U = 0 and 10, T0 = 1 and T0 > receptive field, ragged
  lengths, chunks of 1 frame, of random sizes, and a first chunk shorter than the warm-up;
* the ``_at`` entry points reject inconsistent windows (and positions past 2^31) before touching a device;
* the modified decode kernels compile with the register and spill counts of ptxas recorded below."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import wavenet_oracle as O
from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets.wavenet import decode_window


def _chunked(cfg, p, x, h, totals, mode, uniforms, schedule):
    """oracle decoding through decode_window: one 'call' per chunk; returns per-utterance samples (batch order)"""
    B, T0 = x.shape
    P = max(T0, cfg.receptive_field)
    n_pad, U, ks, Q = P - T0, cfg.upsampling_factor, cfg.kernel_size, cfg.n_quantize
    Uc = max(U, 1)
    dtype = p["causal.conv.weight"].dtype
    st = O.FifoState(cfg, B, dtype)
    carry = {c: np.full(B, Q // 2, np.int64) for c in range(n_pad)}
    carry.update({n_pad + c: x[:, c].astype(np.int64) for c in range(T0)})
    frames, pos, got = 0, 0, [[] for _ in range(B)]
    none = -np.ones(B, dtype=np.int64)
    for F in schedule:
        frames += F
        win = decode_window(pos, frames, P, n_pad, U, ks, totals)
        if win is None:
            continue
        assert win.pos0 == pos and win.n == max(win.counts) and win.end == max(win.pos0, P - 1) + win.n
        # the call sees xs columns >= xs_base and aux frames h_frame0 .. frames - 1 only
        xs = {c: v for c, v in carry.items() if c >= win.xs_base}
        hw = h[:, :, win.h_frame0:frames]
        if U > 0:
            hw = O.upsample(hw, p["upsampling.conv.weight"], p["upsampling.conv.bias"])
        uni = None if uniforms is None else uniforms[:, win.i0:win.i0 + win.n]
        for q in range(win.pos0, win.end):
            prev = [xs[q - (ks - 1 - k)] if q - (ks - 1 - k) >= 0 else none for k in range(ks - 1)]
            col = max(q - n_pad, 0) - win.h_frame0 * Uc
            assert 0 <= col < hw.shape[2], "the window needs an aux column that has not arrived"
            lg = O.fifo_step(cfg, p, st, prev, xs[q], hw[:, :, col].astype(dtype), want_logits=q >= P - 1)
            if lg is not None:
                ic = q - (P - 1) - win.i0
                xs[q + 1] = np.array([O._pick(lg[b], mode, None if uni is None else uni[b][ic]) for b in range(B)])
                for b in range(B):
                    if ic < win.counts[b]:
                        got[b].append(int(xs[q + 1][b]))
        carry, pos = xs, win.end
    assert pos == P - 1 + max(totals)
    return got


def _case(ks, U, long_seed, seed):
    rng = np.random.RandomState(seed)
    cfg = O.Config(32, 5, 8, 12, 3, 2, ks, U)
    p = O.make_params(cfg, seed)
    B = 3
    T0 = cfg.receptive_field + 7 if long_seed else 1
    totals = [int(v) for v in rng.randint(1, 40, size=B)]
    totals[1] = 40
    Uc = max(U, 1)
    nf = (T0 - 1 + max(totals) + Uc - 1) // Uc + 2
    x = rng.randint(0, cfg.n_quantize, size=(B, T0)).astype(np.int64)
    h = rng.standard_normal((B, cfg.n_aux, nf)).astype(np.float32)
    return cfg, p, x, h, totals, nf, rng


def _schedules(nf, rng, rf, Uc):
    ones = [1] * nf
    rand = []
    while sum(rand) < nf:
        rand.append(int(rng.randint(1, 6)))
    short = max(1, (rf - 1) // (2 * Uc))            # first chunk shorter than the warm-up (in samples)
    first_short = [short] + [int(rng.randint(1, 4)) for _ in range(nf)]
    return {"ones": ones, "random": rand, "first_short": first_short}


@pytest.mark.parametrize("ks", [2, 3])
@pytest.mark.parametrize("U", [0, 10])
@pytest.mark.parametrize("long_seed", [False, True])
@pytest.mark.parametrize("mode", ["argmax", "sampling"])
def test_window_reproduces_batch_fast_generate(ks, U, long_seed, mode):
    cfg, p, x, h, totals, nf, rng = _case(ks, U, long_seed, 11 * ks + U + (5 if long_seed else 0))
    uni = rng.uniform(size=(len(totals), max(totals))).astype(np.float32) if mode == "sampling" else None
    outs = O.batch_fast_generate(cfg, p, x, h, totals, mode, None if uni is None else list(uni))
    order = sorted(range(len(totals)), key=lambda b: (totals[b], b))
    want = {b: outs[k].tolist() for k, b in enumerate(order)}
    for name, sched in _schedules(nf, rng, cfg.receptive_field, max(U, 1)).items():
        got = _chunked(cfg, p, x, h, totals, mode, uni, sched)
        for b in range(len(totals)):
            assert got[b] == want[b], (name, b)


def test_window_arithmetic():
    # rf 15, T0 1: P 15, n_pad 14; U 10: frame f covers positions 14 + 10 f .. 14 + 10 f + 9
    assert decode_window(0, 0, 15, 14, 10, 2, [5, 30]) is None
    w = decode_window(0, 1, 15, 14, 10, 2, [5, 30])
    assert (w.pos0, w.end, w.i0, w.n, w.counts, w.xs_base, w.h_frame0) == (0, 24, 0, 10, [5, 10], 0, 0)
    w = decode_window(24, 3, 15, 14, 10, 2, [5, 30])
    assert (w.pos0, w.end, w.i0, w.n, w.counts, w.xs_base, w.h_frame0) == (24, 44, 10, 20, [0, 20], 23, 1)
    # T0 > rf: the warm-up waits for the frames of sample 0 (P = 40, n_pad = 0)
    assert decode_window(0, 3, 40, 0, 10, 3, [8]) is None
    w = decode_window(0, 4, 40, 0, 10, 3, [8])
    assert (w.end, w.n, w.xs_base, w.h_frame0) == (40, 1, 0, 0)
    # sample-rate aux (U = 0)
    w = decode_window(0, 2, 15, 14, 0, 2, [100])
    assert (w.end, w.n) == (16, 2)


def _fake(n):
    return [16 * (k + 1) for k in range(n)]   # non-NULL pointers: the window checks come before any device work


def test_bad_windows_rejected_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)
    seed = ctypes.c_uint64(0)
    # decode_at: (P 4, n_pad 3, U 10, ks 2): xs_base past pos0 - 1, h_frame0 past the frame of pos0, positions past 2^31;
    # (P 10): a window starting inside the warm-up, which no chain of calls produces
    for pos0, xs_base, h_frame0, P, max_n in [(10, 10, 0, 4, 5), (10, 8, 1, 4, 5), (-1, 0, 0, 4, 5),
                                              (0, 0, 0, 2 ** 31 - 10, 100), (2, 1, 0, 10, 5), (8, 7, 0, 10, 5)]:
        rc = lib.wnb_decode_at(*_fake(14), dil, 2, 16, 16, None, None, 2, P, max_n, 3, 4, 256, 28, 32, 64, 512, 2, 10,
                               0, seed, pos0, xs_base, h_frame0, None)
        assert rc == -1 and b"bad window" in lib.wnb_last_error(), (pos0, xs_base, h_frame0)
    rc = lib.wnb_decode_stream_at(*_fake(11), dil, 2, 16, 16, None, None, 2, 4, 5, 3, 4, 256, 28, 32, 64, 512, 2, 10, 0,
                                  seed, 10, 10, 0, None)
    assert rc == -1 and b"bad window" in lib.wnb_last_error()
    rc = lib.wnb_decode_warp_at(*_fake(11), dil, 2, 16, 16, None, None, 2, 4, 5, 3, 4, 28, 10, 0, seed, 16, 2, 10, 10, 0,
                                None)
    assert rc == -1 and b"bad window" in lib.wnb_last_error()
    rc = lib.wnb_decode_bf16_at(*_fake(7), dil, 2, 16, 16, None, None, 2, 4, 5, 3, 4, 256, 28, 32, 512, 256, 2, 10, 0,
                                seed, 10, 10, 0, None)
    assert rc == -1 and b"bad window" in lib.wnb_last_error()


# ptxas -v of every decode instantiation with the window (H100 build flags): (registers, spill stores, spill loads).
# Against the parent: decode<4> 55 -> 64 registers, decode_stream<1> 89 -> 86, decode_bf16<512,256> 231 -> 240,
# decode_bf16<256,256> 171 -> 174; every other count is unchanged, and no spill count changed.
PTXAS = {
    "decode.cu": {"decode_kernelILi1E": (128, 0, 0), "decode_kernelILi2E": (64, 0, 0), "decode_kernelILi4E": (64, 0, 0)},
    "decode_stream.cu": {"decode_stream_kernelILi1E": (86, 0, 0), "decode_stream_kernelILi2E": (80, 0, 0),
                         "decode_stream_kernelILi4E": (104, 0, 0)},
    "decode_warp.cu": {"ILi1ELi16ELb0ELi1E": (93, 0, 0), "ILi1ELi16ELb1ELi1E": (96, 0, 0),
                       "ILi2ELi16ELb0ELi1E": (95, 0, 0), "ILi2ELi16ELb1ELi1E": (96, 12, 12),
                       "ILi4ELi8ELb0ELi1E": (168, 208, 128), "ILi4ELi8ELb1ELi1E": (168, 208, 128),
                       "ILi1ELi16ELb0ELi2E": (127, 0, 0), "ILi1ELi16ELb1ELi2E": (123, 0, 0)},
    "decode_bf16.cu": {"ILi512ELi512E": (255, 0, 0), "ILi512ELi256E": (240, 0, 0), "ILi256ELi256E": (174, 0, 0)},
}


@pytest.mark.parametrize("src", sorted(PTXAS))
def test_decode_kernels_registers_and_spills(src):
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, src),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers", text, re.S):
        found[m.group(1)] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    for key, want in PTXAS[src].items():
        hits = [v for k, v in found.items() if key in k]
        assert hits == [want], (key, hits, found)
