# -*- coding: utf-8 -*-
"""CPU tier: the parallel decode warm-up (``wnb_decode_warp_prefill``, csrc/decode_prefill.cu) without a GPU.

* ``decode_prefill_windows`` against brute-force dependency propagation, and the library's own windows (what the prefill
  launcher uses, layer by layer) and scratch size against it;
* the entry point rejects bad shapes, null pointers and bad dilations before touching a device;
* decode_prefill.cu compiles for sm_90a with the register counts recorded below, no spills and no C7510 note."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets.wavenet import decode_prefill_windows


def _needed(dilations, ks):
    """offsets o >= 1 (position P - 1 - o) at which each layer's input must be known before position P - 1: layer l's
    queue holds its last (ks - 1) d_l inputs, and x_{l+1}(t) reads x_l(t - j d_l), j = 0 .. ks - 1"""
    need = set()
    out = []
    for d in reversed(dilations):
        need = set(range(1, (ks - 1) * d + 1)) | {o + j * d for o in need for j in range(ks)}
        out.append(need)
    return out[::-1]


@pytest.mark.parametrize("ks", [1, 2, 3])
def test_windows_match_dependency_propagation(ks):
    rng = np.random.RandomState(ks)
    cases = [[1, 2, 4, 8] * 3, [1], [512, 1, 2], [2 ** i for i in range(10)]]
    cases += [[int(v) for v in rng.randint(1, 40, size=rng.randint(1, 12))] for _ in range(30)]
    for dil in cases:
        S = decode_prefill_windows(dil, ks)
        assert len(S) == len(dil)
        for l, need in enumerate(_needed(dil, ks)):
            assert need == set(range(1, S[l] + 1)), (dil, ks, l)   # a contiguous window ending at P - 2
        # the windows the prefill launcher and the workspace size use
        out = (ctypes.c_int64 * len(dil))()
        assert _lib.load().wnb_decode_prefill_windows((ctypes.c_int32 * len(dil))(*dil), len(dil), ks, out) == 0
        assert list(out) == S, (dil, ks)


def test_workspace_size():
    lib = _lib.load()
    for dil, ks in (([1, 2, 4, 8] * 3, 2), ([2 ** i for i in range(10)] * 3, 2), ([1, 2, 4], 3)):
        S0 = decode_prefill_windows(dil, ks)[0]
        cd = (ctypes.c_int32 * len(dil))(*dil)
        for B, P in ((1, 1), (3, 2), (64, S0 + 1), (64, S0), (5, 80000)):
            want = 2 * B * 64 * min(S0, P - 1) * 4
            assert lib.wnb_decode_prefill_workspace(B, P, 64, ks, cd, len(dil)) == want, (dil, B, P)
    assert lib.wnb_decode_prefill_workspace(0, 10, 64, 2, (ctypes.c_int32 * 1)(1), 1) == 0
    for bad in ((1, 0, 4), (1, -8, 4)):   # a dilation < 1: no size, and the windows are refused
        cd = (ctypes.c_int32 * 3)(*bad)
        assert lib.wnb_decode_prefill_workspace(2, 100, 64, 2, cd, 3) == 0, bad
        assert lib.wnb_decode_prefill_windows(cd, 3, 2, (ctypes.c_int64 * 3)()) == -1, bad
        assert b"dilations must be >= 1" in lib.wnb_last_error()


def _fake(n):
    return [16 * (k + 1) for k in range(n)]   # non-NULL pointers: every check comes before any device work


def test_bad_arguments_rejected_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)

    def call(ptrs=None, dl=dil, L=2, queues=16, scratch=16, B=2, P=8, n_pad=3, Th=4, A=28, U=10, CL=1):
        return lib.wnb_decode_warp_prefill(*(ptrs or _fake(10)), dl, L, queues, scratch, B, P, n_pad, Th, A, U, CL, None)

    for kw in (dict(B=0), dict(P=0), dict(n_pad=8), dict(n_pad=-1), dict(Th=0), dict(A=0), dict(A=33), dict(U=-1),
               dict(L=0), dict(L=65), dict(CL=0), dict(CL=3)):
        assert call(**kw) == -1 and b"bad shape" in lib.wnb_last_error(), kw
    for i in range(10):
        if i in (2, 3):   # up_w / up_b: needed with U > 0 only
            continue
        ptrs = _fake(10)
        ptrs[i] = None
        assert call(ptrs) == -1 and b"null pointer" in lib.wnb_last_error(), i
    assert call(dl=None) == -1 and b"null pointer" in lib.wnb_last_error()
    assert call(queues=None) == -1 and b"null pointer" in lib.wnb_last_error()
    ptrs = _fake(10)
    ptrs[2] = None
    assert call(ptrs) == -1 and b"upsampling" in lib.wnb_last_error()
    assert call(dl=(ctypes.c_int32 * 2)(1, 3)) == -1 and b"powers of two" in lib.wnb_last_error()
    assert call(dl=(ctypes.c_int32 * 2)(1, 0)) == -1 and b"powers of two" in lib.wnb_last_error()
    assert call(scratch=None) == -1 and b"null scratch" in lib.wnb_last_error()
    assert call(scratch=None, P=1, n_pad=0) == 0   # no warm-up position: nothing to do, no scratch needed


# ptxas -v of decode_prefill.cu (H100 build flags): (registers, spill stores, spill loads)
PTXAS = {"prefill_layer_kernel": (150, 0, 0), "prefill_front_kernel": (26, 0, 0)}


def test_prefill_kernels_registers_and_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "decode_prefill.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    assert "C7510" not in text, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers", text, re.S):
        found[m.group(1)] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    assert len(found) == len(PTXAS), found
    for key, want in PTXAS.items():
        hits = [v for k, v in found.items() if key in k]
        assert hits == [want], (key, hits, found)
