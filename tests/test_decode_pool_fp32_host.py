# -*- coding: utf-8 -*-
"""CPU tier: the host side of decode pools on the fp32 warp decoder.

``wnb_decode_pool_move`` refuses every bad argument before any device work and compiles without spills; a numpy
restatement of its move (a per-layer roll of each slot range) agrees with the header's slot formula for rotations of both
signs and beyond one queue length; the pool's launch form comes from ``wnb_decode_warp_form``; the step counter of an
fp32 pool stays at or above its longest queue, through rebases; and ``bin/decode.py`` refuses ``--pool_capacity`` below
0, or together with ``--chunk_frames``, before it creates the output directory."""
import ctypes
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets import wavenet as W


def move_reference(block, rotation, dilations, ks):
    """One queue block ``[sum_l (ks-1) d_l slots][R]`` moved with ``rotation``: each layer's slot range rolled."""
    out, s0 = np.empty_like(block), 0
    for d in dilations:
        q = (ks - 1) * d
        out[s0:s0 + q] = np.roll(block[s0:s0 + q], rotation, axis=0)
        s0 += q
    return out


@pytest.mark.parametrize("ks", [2, 3])
def test_roll_restatement_matches_the_slot_formula(ks):
    dil = [1, 2, 4, 8, 1, 3]
    nslots = sum((ks - 1) * d for d in dil)
    block = np.arange(nslots * 4, dtype=np.float32).reshape(nslots, 4)
    for rot in (0, 1, -1, 5, -7, 16, -16, 17, -33, 2 ** 31 - 1, -2 ** 31):
        got = move_reference(block, rot, dil, ks)
        s0 = 0
        for d in dil:
            q = (ks - 1) * d
            for s in range(q):   # header: source slot s -> destination slot (s + rotation) mod qlen
                assert np.array_equal(got[s0 + (s + rot) % q], block[s0 + s]), (rot, d, s)
            s0 += q


def _blocks(n, base):
    return (ctypes.c_void_p * max(n, 1))(*[base + 4096 * k for k in range(n)])


def test_move_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)   # 3 slots: 768 bytes at R 64

    def call(src="ok", dst="ok", rot=(-5, 9), n=2, R=64, ks=2, dl=dil, L=2):
        s = _blocks(2, 1 << 20) if src == "ok" else src
        d = _blocks(2, 1 << 24) if dst == "ok" else dst
        r = None if rot is None else (ctypes.c_int32 * max(len(rot), 1))(*rot)
        return lib.wnb_decode_pool_move(s, d, r, n, R, ks, dl, L, None)

    def fails(what, **kw):
        assert call(**kw) == -1, kw
        err = lib.wnb_last_error()
        assert b"decode_pool_move" in err and what in err, (kw, err)

    for kw in (dict(n=0), dict(n=65), dict(n=-1), dict(R=0), dict(R=66), dict(ks=1), dict(L=0), dict(L=65)):
        fails(b"bad shape", **kw)
    for kw in (dict(src=None), dict(dst=None), dict(rot=None), dict(dl=None),
               dict(src=(ctypes.c_void_p * 2)(1 << 20, None)), dict(dst=(ctypes.c_void_p * 2)(None, 1 << 24))):
        fails(b"null pointer", **kw)
    fails(b"not 16-byte aligned", src=(ctypes.c_void_p * 2)(1 << 20, (1 << 20) + 4104))
    fails(b"not 16-byte aligned", dst=(ctypes.c_void_p * 2)((1 << 24) + 8, 1 << 25))
    fails(b"dilations must be positive", dl=(ctypes.c_int32 * 2)(1, 0))
    fails(b"given twice", dst=(ctypes.c_void_p * 2)(1 << 24, 1 << 24))
    fails(b"given twice", dst=(ctypes.c_void_p * 2)(1 << 24, (1 << 24) + 752))        # overlapping blocks
    fails(b"overlaps source", dst=(ctypes.c_void_p * 2)(1 << 24, 1 << 20))            # in place
    fails(b"overlaps source", dst=(ctypes.c_void_p * 2)((1 << 20) + 4096, 1 << 24))   # another block's source
    fails(b"overlaps source", dst=(ctypes.c_void_p * 2)((1 << 20) - 752, 1 << 24))


def test_move_kernel_compiles_without_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    assert "decode_pool.cu" in build.SOURCES
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "decode_pool.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, re.S):
        found[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert len(found) == 1 and all("pool_move_kernel" in k for k in found), found
    assert all(v == (0, 0) for v in found.values()), found


def test_pool_form_is_the_librarys():
    """warp_pool_form returns wnb_decode_warp_form's (NU, W, CL) at every capacity up to past the NU 4 threshold, and
    the thresholds fall where the library puts them: CL 2 up to some S rows, then NU 1, NU 2 and NU 4 ranges of S, 2 S
    and 4 S rows."""
    lib = _lib.load()
    net = W.WaveNet(256, 28, 64, 512, 10, 3, 2, 80)
    L = len(net.dilations)
    forms = []
    for cap in range(1, 700):
        f = (ctypes.c_int32 * 4)()
        assert lib.wnb_decode_warp_form(cap, L, f) == 0
        assert W.warp_pool_form(net, cap) == (f[0], f[1], f[2]), cap
        assert lib.wnb_decode_warp_plan(cap) == f[1] and lib.wnb_decode_warp_cluster(cap) == f[2]
        forms.append((f[0], f[1], f[2]))
    half = max(c for c in range(1, 700) if forms[c - 1][2] == 2)
    sms = 2 * half
    assert all(forms[c - 1] == (1, 16, 2) for c in range(1, half + 1))
    assert all(forms[c - 1] == (1, 16, 1) for c in range(half + 1, sms + 1))
    assert all(forms[c - 1] == (2, 16, 1) for c in range(sms + 1, 2 * sms + 1))
    assert all(forms[c - 1] == (4, 8, 1) for c in range(2 * sms + 1, 700))


def test_pool_form_refuses_other_shapes():
    for args in [(256, 28, 256, 256, 4, 2, 2, 4),    # 256/256: the bf16 decoder's
                 (256, 28, 64, 512, 3, 1, 3, 4),     # ks 3
                 (256, 40, 64, 512, 3, 1, 2, 4),     # n_aux above 32
                 (128, 28, 64, 512, 3, 1, 2, 4)]:    # Q 128
        with pytest.raises(_lib.WnbError, match="warp decoder"):
            W.warp_pool_form(W.WaveNet(*args), 8)


def test_fp32_schedule_counter_stays_above_the_longest_queue(monkeypatch):
    dil = [1, 2, 4, 8] * 2
    monkeypatch.setattr(W, "POOL_COUNTER_LIMIT", 8 + 8 + 40)
    s = W.PoolSchedule(2, 16, dil, 2, 0, g_base=8)
    assert s.g == 8
    for k in range(3):
        s.add(k, 1, 90)
        s.streams[k].frames = 200
    g0s = []
    while True:
        call = s.next_call(7)
        if call is None:
            break
        g0s.append(call.g0)
    assert min(g0s) >= 8 and any(b < a for a, b in zip(g0s, g0s[1:])), g0s
    assert W.PoolSchedule(2, 16, dil, 2, 0).g == 1                     # default: ks - 1, as before
    with pytest.raises(ValueError):
        W.PoolSchedule(2, 16, dil, 3, 0, g_base=1)


@pytest.mark.parametrize("extra", [["--pool_capacity", "-1"], ["--pool_capacity", "4", "--chunk_frames", "7"]])
def test_cli_refuses_before_writing(tmp_path, extra):
    out = tmp_path / "out"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.decode", "--feats", str(tmp_path),
                        "--checkpoint", str(tmp_path / "missing.pkl"), "--outdir", str(out)] + extra,
                       cwd=root, env=dict(os.environ, PYTHONPATH=root), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=300)
    text = r.stdout.decode()
    assert r.returncode == 1, text
    assert "--pool_capacity" in text.splitlines()[-1], text
    assert not out.exists()
