# -*- coding: utf-8 -*-
"""CPU tier: mel-cepstral distortion (csrc/distortion.cu, utils/distortion.py, bin/calc_mcd.py) without a GPU.

The float64 restatement the GPU tier compares against (tests/distortion_reference.py) is pinned by what MCD and DTW
are: identical inputs give 0 and the diagonal path; aligned MCD is symmetric; a sequence against a copy with repeated
frames gives 0 along the expected staircase; hand-built ties follow the tie rule; every matrix up to 6 x 6 agrees with
an exhaustive search over all monotone paths.  Also: the launchers refuse bad arguments before any device work, the
workspace size follows the header's layout, batches split under a workspace budget, the CLI pairs files and refuses
mismatches before computing anything, and distortion.cu compiles for sm_90a without spills."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.bin import calc_mcd
from pytorchwavenetvocoder_b200.utils import distortion as DI
from tests import distortion_reference as R


def test_k_is_the_rounded_product():
    assert DI.K == float(np.float64(10.0) / np.log(np.float64(10.0))) * float(np.sqrt(np.float64(2.0)))
    assert abs(DI.K - 6.141851463713754) < 1e-14


@pytest.mark.parametrize("T", [1, 31, 32, 33, 200])
def test_identical_inputs_give_zero_and_the_diagonal(T):
    a = np.random.RandomState(T).randn(T, 25).astype(np.float32)
    assert R.aligned(a, a) == (0.0, T)
    s, path = R.dtw(a, a)
    assert s == 0.0 and np.array_equal(path, np.stack([np.arange(T)] * 2, axis=1))


def test_c0_is_left_out():
    a = np.random.RandomState(1).randn(40, 25).astype(np.float32)
    b = a.copy()
    b[:, 0] += 3.0
    assert R.aligned(a, b)[0] == 0.0 and R.dtw(a, b)[0] == 0.0


@pytest.mark.parametrize("Tr,Td", [(50, 50), (50, 70), (97, 33), (1, 5)])
def test_aligned_is_symmetric(Tr, Td):
    rng = np.random.RandomState(Tr * Td)
    a, b = rng.randn(Tr, 25).astype(np.float32), rng.randn(Td, 25).astype(np.float32)
    assert R.aligned(a, b) == R.aligned(b, a)
    n = min(Tr, Td)
    assert abs(R.aligned(a, b)[0] - np.sqrt(((a[:n, 1:].astype(float) - b[:n, 1:]) ** 2).sum(1)).sum()) < 1e-9 * n


def test_repeated_frames_give_zero_along_the_staircase():
    rng = np.random.RandomState(3)
    ref = rng.randn(40, 25).astype(np.float32)
    reps = rng.randint(1, 4, size=40)
    dec = np.repeat(ref, reps, axis=0)
    s, path = R.dtw(ref, dec)
    assert s == 0.0
    assert np.array_equal(path, np.stack([np.repeat(np.arange(40), reps), np.arange(len(dec))], axis=1))
    s, path = R.dtw(dec, ref)      # the other way round: the path runs down the columns
    assert s == 0.0
    assert np.array_equal(path, np.stack([np.arange(len(dec)), np.repeat(np.arange(40), reps)], axis=1))


def test_tie_rule():
    # all three predecessors tie: the diagonal
    assert np.array_equal(R.dtw(None, None, dist=np.zeros((2, 2)))[1], [[0, 0], [1, 1]])
    # (i-1, j) and (i, j-1) tie below the diagonal: (i-1, j); and at (1, 2) the diagonal ties with (i-1, j)
    d = np.array([[0, 0, 0], [0, 5, 0], [0, 0, 0]], dtype=float)
    assert np.array_equal(R.dtw(None, None, dist=d)[1], [[0, 0], [0, 1], [1, 2], [2, 2]])
    # the diagonal ties with (i, j-1), and with (i-1, j): the diagonal
    d = np.array([[0, 1], [0, 0]], dtype=float)
    assert np.array_equal(R.dtw(None, None, dist=d)[1], [[0, 0], [1, 1]])
    d = np.array([[0, 0, 0], [1, 1, 0]], dtype=float)
    assert np.array_equal(R.dtw(None, None, dist=d)[1], [[0, 0], [0, 1], [1, 2]])
    # column 0 has one predecessor, (i-1, 0)
    d = np.array([[0, 1], [0, 1], [1, 0]], dtype=float)
    assert np.array_equal(R.dtw(None, None, dist=d)[1], [[0, 0], [1, 0], [2, 1]])
    # the same ties from frames: integer cepstra (D = 1), distances |a - b|
    ref = np.array([[9, 0], [9, 1], [9, 0]], dtype=np.float32)
    dec = np.array([[7, 0], [7, 1], [7, 1], [7, 0]], dtype=np.float32)
    s, path = R.dtw(ref, dec)
    assert s == 0.0 and np.array_equal(path, [[0, 0], [1, 1], [1, 2], [2, 3]])


@pytest.mark.parametrize("Tr", range(1, 7))
@pytest.mark.parametrize("Td", range(1, 7))
def test_restatement_agrees_with_exhaustive_search(Tr, Td):
    rng = np.random.RandomState(100 * Tr + Td)
    ref, dec = rng.randn(Tr, 4).astype(np.float32), rng.randn(Td, 4).astype(np.float32)
    s, path = R.dtw(ref, dec)
    least, paths = R.dtw_brute(R.dist_matrix(ref, dec))
    assert s == least and len(paths) == 1 and np.array_equal(path, paths[0])
    assert R.path_sum(ref, dec, path) == s
    # integer distances: many ties; the cost is the least and the path is one of the cheapest
    dist = rng.randint(0, 3, size=(Tr, Td)).astype(float)
    s, path = R.dtw(None, None, dist=dist)
    least, paths = R.dtw_brute(dist)
    assert s == least and any(np.array_equal(path, p) for p in paths)
    steps = {tuple(x) for x in path[1:] - path[:-1]}
    assert steps <= {(1, 1), (1, 0), (0, 1)} and tuple(path[0]) == (0, 0) and tuple(path[-1]) == (Tr - 1, Td - 1)


def test_butterfly_is_the_lane_tree():
    v = np.random.RandomState(5).randn(32)
    lanes = [list(v)]
    for o in (16, 8, 4, 2, 1):
        prev = lanes[-1]
        lanes.append([prev[l] + prev[l ^ o] for l in range(32)])
    assert R.butterfly32(v) == lanes[-1][0]


# ---- the library: arguments, workspace, launch groups (no device work) ------------------------------------------------

def _offs(*lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def test_launchers_refuse_before_device_work():
    lib = _lib.load()
    ok_r, ok_d = _offs(5, 7), _offs(6, 3)

    def aligned(n_cols=25, r=ok_r, d=ok_d, n=2, ptrs=1):
        return lib.wnb_mcd_aligned(ptrs and 256, ptrs and 512, n_cols, ptrs and 1024, 2048, r.ctypes.data,
                                   d.ctypes.data, n, 4096, 8192, None)

    def dtw(n_cols=25, r=ok_r, d=ok_d, n=2, ws=1 << 20, ws_bytes=1 << 30, path=None):
        return lib.wnb_mcd_dtw(256, 512, n_cols, 1024, 2048, r.ctypes.data, d.ctypes.data, n, ws, ws_bytes, 4096,
                               8192, path, None)

    for call in (aligned, dtw):
        for kw, rc, what in ((dict(n_cols=42), -3, b"columns is not supported"), (dict(n_cols=1), -3, b"columns"),
                             (dict(r=_offs(5, 0)), -3, b"pair 1 has 0 reference"),
                             (dict(d=_offs(0, 2)), -3, b"pair 0 has 5 reference and 0 decoded"),
                             (dict(n=0), -1, b"n_pairs > 0")):
            assert call(**kw) == rc, (call, kw)
            assert what in lib.wnb_last_error(), (kw, lib.wnb_last_error())
    assert aligned(ptrs=0) == -1 and b"null pointer" in lib.wnb_last_error()
    assert dtw(ws=None) == -1 and b"null pointer" in lib.wnb_last_error()
    assert dtw(ws=(1 << 20) + 8) == -1 and b"16-byte" in lib.wnb_last_error()
    assert dtw(path=4100) == -1 and b"8-byte" in lib.wnb_last_error()
    need = DI.dtw_workspace_bytes(5, 6) + DI.dtw_workspace_bytes(7, 3)
    assert dtw(ws_bytes=need - 1) == -1 and b"workspace bytes" in lib.wnb_last_error()


def test_workspace_follows_the_header_layout():
    B, S = 256, 4096
    a16 = lambda v: (v + 15) // 16 * 16  # noqa: E731
    for tr, td in ((1, 1), (255, 3), (256, 3), (257, 3), (2000, 2000), (3, S), (3, S + 1), (513, 9000)):
        want = a16(-(-tr // B) * B * (td + B - 1)) + (a16(8 * td) if td > S else 0)
        assert DI.dtw_workspace_bytes(tr, td) == want, (tr, td)
    assert DI.dtw_workspace_bytes(0, 5) == 0 and DI.dtw_workspace_bytes(5, 0) == 0
    assert DI.dtw_workspace_bytes(1 << 24, 1) > 0 and DI.dtw_workspace_bytes((1 << 24) + 1, 1) == 0


def test_launch_groups_split_under_the_budget():
    lens_r, lens_d = [300, 10, 600, 5, 5, 4000], [200, 10, 700, 5, 6, 100]
    need = [DI.dtw_workspace_bytes(a, b) for a, b in zip(lens_r, lens_d)]
    assert DI.launch_groups(lens_r, lens_d, 1 << 40) == [(0, 6, sum(need))]
    budget = need[0] + need[1]
    groups = DI.launch_groups(lens_r, lens_d, budget)
    assert [g[:2] for g in groups][0] == (0, 2) and groups[0][2] == budget
    assert sum(b - a for a, b, _ in groups) == 6 and all(g[0] == h[1] for g, h in zip(groups[1:], groups))
    for a, b, used in groups:      # each fits, or is one pair that alone needs more
        assert used == sum(need[a:b]) and (used <= budget or b - a == 1)
    assert DI.launch_groups(lens_r, lens_d, 1) == [(p, p + 1, need[p]) for p in range(6)]


def test_mcd_batch_refuses_mismatched_inputs():
    a = np.zeros((4, 25), np.float32)
    with pytest.raises(ValueError, match="2 reference and 1 decoded"):
        DI.mcd_batch([a, a], [a])
    with pytest.raises(ValueError, match="same number of coefficients"):
        DI.mcd_batch([a], [np.zeros((4, 26), np.float32)])
    with pytest.raises(ValueError, match="non-empty"):
        DI.mcd_batch([a], [np.zeros((0, 25), np.float32)])
    with pytest.raises(ValueError, match="paths come from DTW"):
        DI.mcd_batch([a], [a], return_path=True)
    r = DI.mcd_batch([], [])
    assert len(r.mcd) == 0 and np.isnan(DI.corpus_mcd(r)[0])


def test_corpus_mcd_is_frame_weighted():
    r = DI.Mcd(np.array([DI.K * 3.0 / 3, DI.K * 10.0 / 1]), np.array([3, 1]), np.array([3.0, 10.0]), None)
    corpus, mean = DI.corpus_mcd(r)
    assert corpus == DI.K * 13.0 / 4 and mean == (r.mcd[0] + r.mcd[1]) / 2


# ---- the CLI: pairing and refusals ------------------------------------------------------------------------------------

def test_pair_files_by_basename():
    pairs, errors = calc_mcd.pair_files(["n/a.wav", "n/b.wav", "n/c.wav"], ["d/c.wav", "d/a.wav", "d/b.wav"])
    assert errors == [] and pairs == [("a", "n/a.wav", "d/a.wav"), ("b", "n/b.wav", "d/b.wav"),
                                      ("c", "n/c.wav", "d/c.wav")]
    pairs, errors = calc_mcd.pair_files(["n/a.wav", "n/b.wav"], ["d/a.wav", "d/x.wav"])
    assert pairs == [("a", "n/a.wav", "d/a.wav")]
    assert any("n/b.wav has no decoded counterpart" in e for e in errors)
    assert any("d/x.wav has no reference counterpart" in e for e in errors)
    _, errors = calc_mcd.pair_files(["n/a.wav", "m/a.wav"], ["d/a.wav"])
    assert errors == ["reference wavs n/a.wav and m/a.wav have the same basename"]


def test_check_pairs():
    info = {"r1": (16000, 16000), "d1": (16000, 16000 + 160), "d2": (16000, 16000 + 240), "d3": (22050, 16000),
            "d4": (16000, 1023), "r4": (16000, 1024)}
    pairs = [("u", "r1", "d1")]
    assert calc_mcd.check_pairs(pairs, info.get, 16000, 1024, 80, 2, False) == []
    errs = calc_mcd.check_pairs([("u", "r1", "d2")], info.get, 16000, 1024, 80, 2, False)
    assert len(errs) == 1 and "r1 has 188 frames and d2 has 191" in errs[0] and "--dtw" in errs[0]
    assert calc_mcd.check_pairs([("u", "r1", "d2")], info.get, 16000, 1024, 80, 3, False) == []
    assert calc_mcd.check_pairs([("u", "r1", "d2")], info.get, 16000, 1024, 80, 2, True) == []
    errs = calc_mcd.check_pairs([("u", "r1", "d3")], info.get, 16000, 1024, 80, 2, True)
    assert errs == ["d3 is sampled at 22050 Hz, not --fs 16000"]
    errs = calc_mcd.check_pairs([("u", "r4", "d4")], info.get, 16000, 1024, 80, 2, True)
    assert errs == ["d4 has 1023 samples, fewer than --fftl 1024, so it has no frames"]


def _write(path, fs, n, seed=0):
    from scipy.io import wavfile
    wavfile.write(path, fs, np.int16(np.random.RandomState(seed).randn(n) * 1000))


@pytest.mark.parametrize("case", ["unpaired", "rate", "short", "frames"])
def test_cli_refuses_before_computing(tmp_path, caplog, case):
    ref, dec = tmp_path / "ref", tmp_path / "dec"
    ref.mkdir()
    dec.mkdir()
    _write(str(ref / "a.wav"), 16000, 4000)
    n_dec = {"frames": 4400, "short": 1000}.get(case, 4000)
    _write(str(dec / "a.wav"), 22050 if case == "rate" else 16000, n_dec)
    if case == "unpaired":
        _write(str(ref / "b.wav"), 16000, 4000)
    out = tmp_path / "mcd.tsv"
    with pytest.raises(SystemExit) as e:
        calc_mcd.main(["--reference", str(ref), "--decoded", str(dec), "--outfile", str(out)])
    assert e.value.code == 1 and not out.exists()
    text = caplog.text
    want = {"unpaired": "b.wav has no decoded counterpart", "rate": "sampled at 22050 Hz",
            "short": "fewer than --fftl 1024", "frames": "compare them along a time-warping path with --dtw"}[case]
    assert want in text and "nothing was computed" in text
    assert str(dec / "a.wav") in text or str(ref / "b.wav") in text


def test_distortion_kernels_compile_without_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    assert "distortion.cu" in build.SOURCES
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "distortion.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, re.S):
        found[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert sorted(k for k in found) == sorted(k for k in found if "mcd_" in k) and len(found) == 2, found
    assert all(v == (0, 0) for v in found.values()), found
