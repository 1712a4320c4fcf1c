# -*- coding: utf-8 -*-
"""CPU tier: the parallel warm-up of the bf16 decoder (``wnb_decode_bf16_prefill``, csrc/decode_bf16_prefill.cu) without
a GPU.

* the scratch size against the formula counted from shapes (fp32 + bf16 x_l and bf16 z over the largest pruned window);
* the entry point rejects bad shapes, null pointers, bad dilations and uncovered shapes before touching a device;
* decode_bf16_prefill.cu compiles for sm_90a with the register counts recorded below, no spills and no C7510 / C7513
  note (a serialised wgmma)."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets.wavenet import decode_prefill_windows

ARCTIC_DIL = [2 ** i for i in range(10)] * 3


def test_workspace_size():
    lib = _lib.load()
    for dil, ks, R in ((ARCTIC_DIL, 2, 512), ([2 ** i for i in range(10)], 3, 512), ([1, 2, 4, 8], 2, 256)):
        S0 = decode_prefill_windows(dil, ks)[0]
        cd = (ctypes.c_int32 * len(dil))(*dil)
        for B, P in ((1, 1), (3, 2), (64, S0 + 1), (64, S0), (70, 80000)):
            want = B * min(S0, P - 1) * R * (4 + 2 + 2)
            assert lib.wnb_decode_bf16_prefill_workspace(B, P, R, ks, cd, len(dil)) == want, (dil, B, P)
    # arctic, B = 64, one-sample seed: 64 x 3069 positions x 512 channels x 8 bytes
    assert lib.wnb_decode_bf16_prefill_workspace(64, 3070, 512, 2, (ctypes.c_int32 * 30)(*ARCTIC_DIL), 30) == \
        64 * 3069 * 512 * 8
    assert lib.wnb_decode_bf16_prefill_workspace(0, 10, 512, 2, (ctypes.c_int32 * 1)(1), 1) == 0
    assert lib.wnb_decode_bf16_prefill_workspace(1, 10, 512, 2, (ctypes.c_int32 * 1)(1), 65) == 0
    for bad in ((1, 0, 4), (1, -8, 4)):
        assert lib.wnb_decode_bf16_prefill_workspace(2, 100, 512, 2, (ctypes.c_int32 * 3)(*bad), 3) == 0, bad


def _fake(n):
    return [16 * (k + 1) for k in range(n)]   # non-NULL pointers: every check comes before any device work


def test_bad_arguments_rejected_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)

    def call(ptrs=None, dl=dil, L=2, queues=16, scratch=16, B=2, P=8, n_pad=3, Th=4, A=28, Ap=32, R=512, S=256, ks=2,
             U=10):
        return lib.wnb_decode_bf16_prefill(*(ptrs or _fake(7)), dl, L, queues, scratch, B, P, n_pad, Th, A, Ap, R, S, ks,
                                           U, None)

    for kw in (dict(B=0), dict(P=0), dict(n_pad=8), dict(n_pad=-1), dict(Th=0), dict(A=0), dict(Ap=16), dict(R=0),
               dict(S=0), dict(ks=0), dict(U=-1), dict(L=0)):
        assert call(**kw) == -1 and b"bad shape" in lib.wnb_last_error(), kw
    for i in range(7):
        if i in (2, 3):   # up_w / up_b: needed with U > 0 only
            continue
        ptrs = _fake(7)
        ptrs[i] = None
        assert call(ptrs) == -1 and b"null pointer" in lib.wnb_last_error(), i
    assert call(dl=None) == -1 and b"null pointer" in lib.wnb_last_error()
    assert call(queues=None) == -1 and b"null pointer" in lib.wnb_last_error()
    ptrs = _fake(7)
    ptrs[2] = None
    assert call(ptrs) == -1 and b"upsampling" in lib.wnb_last_error()
    # shapes the bf16 decoder does not cover: WNB_ERR_UNSUPPORTED
    for kw in (dict(R=64, S=512), dict(R=512, S=128), dict(ks=4), dict(ks=1), dict(Ap=40, A=40), dict(L=65)):
        assert call(**kw) == -3 and b"not covered" in lib.wnb_last_error(), kw
    assert call(dl=(ctypes.c_int32 * 2)(1, 0)) == -1 and b"dilations must be positive" in lib.wnb_last_error()
    assert call(scratch=None) == -1 and b"null scratch" in lib.wnb_last_error()


# ptxas -v of decode_bf16_prefill.cu (H100 build flags): (registers, spill stores, spill loads)
PTXAS = {"prefill_gate_kernelILi512E": (144, 0, 0), "prefill_gate_kernelILi256E": (88, 0, 0),
         "prefill_res_kernelILi512ELi512E": (140, 0, 0), "prefill_res_kernelILi512ELi256E": (124, 0, 0),
         "prefill_res_kernelILi256ELi256E": (80, 0, 0),
         "prefill_front_kernelILi512E": (34, 0, 0), "prefill_front_kernelILi256E": (34, 0, 0)}


def test_prefill_kernels_registers_and_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin",
                                             os.path.join(build.CSRC, "decode_bf16_prefill.cu"),
                                             "-o", os.path.join(tmp, "d.cubin")],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    assert not [line for line in text.splitlines() if "C7510" in line or "C7513" in line], text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers", text, re.S):
        found[m.group(1)] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    assert len(found) == len(PTXAS), found
    for key, want in PTXAS.items():
        hits = [v for k, v in found.items() if key in k]
        assert hits == [want], (key, hits, found)
