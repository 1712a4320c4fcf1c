# -*- coding: utf-8 -*-
"""CPU tier: the streaming decoder's coverage query, the pool's kernel selection, the argument checks of
``wnb_decode_stream_prefill`` and the ptxas counts of its kernels.

* ``wnb_decode_stream_supported`` equals a Python restatement of the launcher's width and shared-memory rule over a
  grid of shapes (and, by construction, the launcher uses the same host function);
* ``pool_kernel``: "auto" follows ``decode_math``, a named kernel must belong to it, unknown names are refused;
* the prefill refuses bad shapes, null pointers and dilations < 1 before any device work, reports an uncovered shape as
  unsupported, and needs no scratch when there is no queued warm-up position."""
import ctypes
import itertools
import os
import re
import subprocess
import tempfile

import pytest

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets import wavenet as W


def _r4(v):
    return (v + 3) & ~3


def _stream_plan(Q, Ap, R, S, ks, L, NU=1):
    """decode_stream.cu's stream_plan, restated: (NU, ring slots) for a launch that starts at ``NU`` utterances per CTA
    (1 at B <= SMs, 2 at B <= 2 SMs, else 4), or None when the shape is not covered"""
    widths = [_r4(2 * R), _r4(R), _r4(S), _r4(S), _r4(Q)]
    if any(w // 4 > 256 or w * 4 > 32 * 1024 for w in widths):
        return None
    if L > 64 or R % 4 or S % 4 or Ap % 4:
        return None
    K1 = ks * R + Ap
    while True:
        work = 4 * NU * (K1 + 2 * R + 2 * S + _r4(Q) + Ap + (ks - 1) * L * R + 1024)
        nslot = 0 if work + 2 * 32 * 1024 + 512 > 227 * 1024 else min((227 * 1024 - 64 - work - 256) // (32 * 1024), 6)
        if nslot >= 2 or NU == 1:
            break
        NU //= 2
    return (NU, nslot) if nslot >= 2 else None


def _supported(Q, Ap, R, S, ks, L):
    """decode_stream.cu's coverage query: stream_plan at NU = 1"""
    return _stream_plan(Q, Ap, R, S, ks, L) is not None


def test_supported_matches_the_launch_rule():
    lib = _lib.load()
    n = 0
    for Q, Ap, R, S, ks, L in itertools.product((64, 256, 1022, 1024, 1028), (32, 34, 80, 256, 512), (4, 64, 256, 510,
                                                512, 516), (62, 64, 256, 512, 1024, 1028), (1, 2, 3, 5),
                                                (1, 10, 30, 64, 65)):
        want = _supported(Q, Ap, R, S, ks, L)
        assert bool(lib.wnb_decode_stream_supported(Q, Ap, R, S, ks, L)) == want, (Q, Ap, R, S, ks, L)
        n += want
    assert n > 1000   # the grid reaches both sides of every condition
    assert lib.wnb_decode_stream_supported(256, 32, 512, 256, 2, 30)      # arctic 512/256
    assert lib.wnb_decode_stream_supported(256, 96, 512, 256, 3, 30)      # ljspeech-melspc (n_aux 80)
    assert not lib.wnb_decode_stream_supported(256, 32, 512, 256, 2, 65)


def test_pool_kernel_selection():
    assert W.pool_kernel("fp32", "auto") == "warp"
    assert W.pool_kernel("bf16", "auto") == "bf16"
    assert W.pool_kernel("fp32", "stream") == "stream"
    assert W.pool_kernel("fp32", "warp") == "warp"
    assert W.pool_kernel("bf16", "bf16") == "bf16"
    for math, kernel in (("fp32", "bf16"), ("bf16", "stream"), ("bf16", "warp")):
        with pytest.raises(_lib.WnbError, match="does not run"):
            W.pool_kernel(math, kernel)
    with pytest.raises(_lib.WnbError, match="decode_math"):
        W.pool_kernel("tf32", "auto")
    with pytest.raises(ValueError):
        W.pool_kernel("fp32", "direct")


def _fake(n):
    return [16 * (k + 1) for k in range(n)]   # non-NULL pointers: every check comes before any device work


def test_prefill_bad_arguments_rejected_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 3)

    def call(ptrs=None, dl=dil, L=2, queues=16, scratch=16, B=2, P=8, n_pad=3, Th=4, Q=256, A=28, Ap=32, R=64, S=64,
             ks=3, U=10):
        return lib.wnb_decode_stream_prefill(*(ptrs or _fake(9)), dl, L, queues, scratch, B, P, n_pad, Th, Q, A, Ap, R,
                                             S, ks, U, None)

    for kw in (dict(B=0), dict(P=0), dict(n_pad=8), dict(n_pad=-1), dict(Th=0), dict(Q=0), dict(A=0), dict(Ap=24),
               dict(R=0), dict(S=0), dict(ks=0), dict(U=-1), dict(L=0)):
        assert call(**kw) == -1 and b"bad shape" in lib.wnb_last_error(), kw
    for i in range(9):
        if i in (2, 3):   # up_w / up_b: needed with U > 0 only
            continue
        ptrs = _fake(9)
        ptrs[i] = None
        assert call(ptrs) == -1 and b"null pointer" in lib.wnb_last_error(), i
    assert call(dl=None) == -1 and b"null pointer" in lib.wnb_last_error()
    assert call(queues=None) == -1 and b"null pointer" in lib.wnb_last_error()
    ptrs = _fake(9)
    ptrs[2] = None
    assert call(ptrs) == -1 and b"upsampling" in lib.wnb_last_error()
    assert call(dl=(ctypes.c_int32 * 2)(1, 0)) == -1 and b">= 1" in lib.wnb_last_error()
    assert call(S=62) == -3 and b"not covered" in lib.wnb_last_error()     # outside the streaming kernel
    assert call(R=1024) == -3 and b"not covered" in lib.wnb_last_error()
    assert call(L=65, dl=(ctypes.c_int32 * 65)(*[1] * 65)) == -3
    assert call(scratch=None) == -1 and b"null scratch" in lib.wnb_last_error()
    assert call(scratch=None, P=1, n_pad=0) == 0   # no warm-up position: nothing to do, no scratch needed
    assert call(scratch=None, queues=None, ks=1) == 0   # ks 1 keeps no queues


def test_prefill_scratch_is_bounded_by_64_rows():
    lib = _lib.load()
    dil = [2 ** i for i in range(10)] * 3
    cd = (ctypes.c_int32 * 30)(*dil)
    rf = sum(dil) + 1
    per_row = lib.wnb_decode_prefill_workspace(1, rf, 512, 2, cd, 30)
    assert per_row == 2 * 512 * (rf - 1) * 4
    assert W.STREAM_PREFILL_ROWS == 64
    assert lib.wnb_decode_prefill_workspace(W.STREAM_PREFILL_ROWS, rf, 512, 2, cd, 30) == 64 * per_row   # ~0.8 GB


# ptxas -v of decode_stream_prefill.cu (H100 build flags): (registers, spill stores, spill loads)
PTXAS = {"stream_prefill_layer_kernel": (118, 0, 0), "stream_prefill_front_kernel": (32, 0, 0)}


def test_prefill_kernels_registers_and_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin",
                                             os.path.join(build.CSRC, "decode_stream_prefill.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers", text, re.S):
        found[m.group(1)] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    assert len(found) == len(PTXAS), found
    for key, want in PTXAS.items():
        hits = [v for k, v in found.items() if key in k]
        assert hits == [want], (key, hits, found)
