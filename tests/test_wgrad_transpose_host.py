# -*- coding: utf-8 -*-
"""CPU tier: the tf32 B transpose of the weight-gradient kernel, as wnb_wgrad_transpose_map reports it from the same
functions the kernel's consumer loop runs.  For every B group count, with and without the all-ones group of a bias
gradient, the 4 x 4 units of one stage move every element of the swizzled B sub-tiles exactly once, to its place in the
K-major 128B-swizzled tile, clear of the ones rows; and every warp-wide 16-byte load and store takes the least number of
shared-memory wavefronts, counted per quarter warp and over the whole warp.  The former mapping (one 16-byte load and
four 4-byte stores per thread) is restated as a control: its stores take 4 wavefronts where 1 would do.

Also compiles wgrad_tc.cu for sm_90a (needs nvcc, not a GPU): neither kernel instantiation spills, and ptxas reports
no serialised or dropped wgmma pipeline (notes C7510, C7512, C7513)."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import pytest

SUB = 32 * 128            # one swizzled [32 time rows x 32 fp32 channels] sub-tile, bytes
CONSUMERS = 256


def sw128(r, c):
    """byte offset of element (row r, column c < 32) of a [rows x 32 fp32] tile in the 128B-swizzled layout"""
    return r * 128 + ((((c >> 2) ^ r) & 7) << 4) + ((c & 3) << 2)


def transpose_map(nB):
    from pytorchwavenetvocoder_b200 import _lib as L_
    lib = L_.load()
    buf = (ctypes.c_int * (640 * nB))()
    n = lib.wnb_wgrad_transpose_map(nB, buf)
    assert n == 64 * nB, lib.wnb_last_error()
    return [tuple(buf[10 * k:10 * k + 10]) for k in range(n)]


def wavefronts(accesses, width, lanes_per_part):
    """Shared-memory wavefronts of one warp-wide access: (lane, byte address) pairs of `width` bytes each.  The warp is
    served `lanes_per_part` lanes at a time; a part takes as many wavefronts as the largest number of distinct 4-byte
    words any one of the 32 banks holds for it."""
    parts = {}
    for lane, a in accesses:
        assert a % width == 0
        parts.setdefault(lane // lanes_per_part, []).append(a)
    total = 0
    for addrs in parts.values():
        banks = {}
        for a in addrs:
            for w in range(a // 4, (a + width) // 4):
                banks.setdefault(w % 32, set()).add(w)
        total += max(len(s) for s in banks.values())
    return total


def least_wavefronts(accesses, width):
    return -(-len(accesses) * width // 128)


def warp_accesses(rows):
    """rows of (thread, iteration, offsets...) -> {(warp, iteration): [(lane, row)]}"""
    out = {}
    for row in rows:
        out.setdefault((row[0] // 32, row[1]), []).append((row[0] % 32, row))
    return out


@pytest.mark.parametrize("ones", [0, 1])
@pytest.mark.parametrize("nB", range(1, 8))
def test_transpose_moves_every_element_to_its_sw128_place(nB, ones):
    rows = transpose_map(nB)
    assert all(0 <= r[0] < CONSUMERS for r in rows)
    where = {}
    for r in rows:
        src, dst = r[2:6], r[6:10]
        for i in range(4):          # load i: time row i of the unit's 4 channels
            for j in range(4):      # store j: channel j of the unit's 4 time rows
                assert src[i] + 4 * j not in where
                where[src[i] + 4 * j] = dst[j] + 4 * i
    expect = {g * SUB + sw128(t, c): sw128(32 * g + c, t) for g in range(nB) for t in range(32) for c in range(32)}
    assert where == expect
    # the transposed rows and the ones rows (32 after them, filled by 16-byte stores) tile [N x 32] exactly once
    N = 32 * (nB + ones)
    written = sorted(list(where.values()) + [32 * nB * 128 + 4 * i for i in range(32 * 32 * ones)])
    assert written == list(range(0, N * 128, 4))


@pytest.mark.parametrize("nB", range(1, 8))
def test_transpose_accesses_take_the_least_wavefronts(nB):
    rows = transpose_map(nB)
    per_thread = {}
    for r in rows:
        per_thread[r[0]] = per_thread.get(r[0], 0) + 1
    assert max(per_thread.values()) == -(-nB // 4)          # a static split: at most one unit more than any other
    for (w, it), acc in warp_accesses(rows).items():
        assert sorted(lane for lane, _ in acc) == list(range(32)), (w, it)   # whole warps
        for i in range(4):
            for col in (2 + i, 6 + i):                       # load i, store i
                a = [(lane, r[col]) for lane, r in acc]
                least = least_wavefronts(a, 16)
                assert wavefronts(a, 16, 8) == least, (nB, w, it, col)      # served a quarter warp at a time
                assert wavefronts(a, 16, 32) == least, (nB, w, it, col)     # served as one warp


def scalar_store_map(nB):
    """The former transpose: float4 piece idx = t + 256 k of the B sub-tiles, time row r, channel chunk c4, one 16-byte
    load and four 4-byte stores (thread, iteration, load offset, 4 store offsets)."""
    rows = []
    for t in range(CONSUMERS):
        for it, idx in enumerate(range(t, nB * 256, CONSUMERS)):
            g, r, c4 = idx >> 8, (idx >> 3) & 31, idx & 7
            rows.append((t, it, g * SUB + r * 128 + ((c4 ^ (r & 7)) << 4))
                        + tuple(sw128(32 * g + 4 * c4 + j, r) for j in range(4)))
    return rows


def test_wavefront_count_sees_the_scalar_store_conflicts():
    for (w, it), acc in warp_accesses(scalar_store_map(6)).items():
        for j in range(4):
            a = [(lane, r[3 + j]) for lane, r in acc]
            assert least_wavefronts(a, 4) == 1
            assert wavefronts(a, 4, 32) == 4


def _nvcc():
    from pytorchwavenetvocoder_b200 import build
    try:
        cand = build._nvcc()
    except RuntimeError:
        return None
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


def test_wgrad_tc_kernels_keep_their_registers_and_async_wgmma():
    from pytorchwavenetvocoder_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "wgrad_tc.cu"),
                                "-o", os.path.join(tmp, "wgrad_tc.cubin")]
        pr = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = pr.stdout.decode()
    assert pr.returncode == 0, text
    spills = re.findall(r"Function properties for (\S*wgrad_tc_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                        r"stores, (\d+) bytes spill loads", text)
    assert len(spills) == 2, text
    assert all(int(s) == 0 and int(l) == 0 for _, s, l in spills), spills
    notes = [line for line in text.splitlines() if re.search(r"C751[023]", line)]
    assert not notes, "\n".join(notes)
