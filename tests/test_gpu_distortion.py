# -*- coding: utf-8 -*-
"""GPU tier: mel-cepstral distortion (wnb_mcd_aligned, wnb_mcd_dtw, utils/distortion.py, bin/calc_mcd.py) bit for bit
against the float64 restatement of tests/distortion_reference.py: the per-pair sums, the counts and the DTW paths are
compared with np.array_equal.  Cases: random and integer-valued (tie-heavy) frames, Tr != Td both ways down to one
frame, lengths on either side of the DTW strip height (WNB_MCD_DTW_THREADS rows) and of the shared-memory row limit
(WNB_MCD_DTW_SMEM_COLS columns), D from 1 to 40, and one batch mixing all of them split over several launches by the
workspace budget; a pair gives the same bits alone as in the batch and on a second run.  The CLI runs end to end on
synthetic wavs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import distortion_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(rng, T, cols, kind):
    if kind == "int":
        return rng.randint(-1, 2, size=(T, cols)).astype(np.float32)
    return (rng.randn(T, cols) * np.linspace(2.0, 0.05, cols)).astype(np.float32)


def _case(seed, Tr, Td, cols=25, kind="rand"):
    rng = np.random.RandomState(seed)
    return _frames(rng, Tr, cols, kind), _frames(rng, Td, cols, kind)


SHAPES = [(1, 1), (1, 7), (7, 1), (1, 300), (300, 1), (40, 57), (57, 40), (255, 255), (256, 256), (257, 255),
          (255, 257), (513, 300), (300, 513), (3, 4096), (3, 4097), (260, 4097), (4097, 3)]


def _check(pairs, dtw, **kw):
    from pytorchwavenetvocoder_b200.utils.distortion import K, mcd_batch
    refs, decs = [p[0] for p in pairs], [p[1] for p in pairs]
    got = mcd_batch(refs, decs, dtw=dtw, return_path=dtw, **kw)
    for k, (a, b) in enumerate(pairs):
        if dtw:
            s, path = R.dtw(a, b)
            assert np.array_equal(got.paths[k], path), (k, a.shape, b.shape)
            n = len(path)
        else:
            s, n = R.aligned(a, b)
        assert np.array_equal(got.sums[k], s), (k, a.shape, b.shape, dtw, got.sums[k], s)
        assert got.counts[k] == n, (k, a.shape, b.shape, dtw)
        assert np.array_equal(got.mcd[k], K * s / n)
    return got


@pytest.mark.parametrize("dtw", [False, True])
@pytest.mark.parametrize("kind", ["rand", "int"])
def test_shapes_bit_exact(dtw, kind):
    pairs = [_case(17 * i + (kind == "int"), Tr, Td, kind=kind) for i, (Tr, Td) in enumerate(SHAPES)]
    _check(pairs, dtw)


@pytest.mark.parametrize("cols", [2, 25, 36, 41])
def test_coefficient_counts(cols):
    pairs = [_case(cols + i, Tr, Td, cols=cols) for i, (Tr, Td) in enumerate([(33, 45), (300, 290), (5, 1)])]
    _check(pairs, False)
    _check(pairs, True)


def test_recipe_length_pair():
    """A 10 s arctic utterance (1 988 frames of order 24) against a 10 % slower copy with noise."""
    rng = np.random.RandomState(7)
    a = _frames(rng, 1988, 25, "rand")
    idx = np.minimum((np.arange(2187) / 1.1).astype(int), 1987)
    b = (a[idx] + rng.randn(2187, 25).astype(np.float32) * 0.05).astype(np.float32)
    _check([(a, b)], True)


def test_split_batch_alone_and_again():
    from pytorchwavenetvocoder_b200.utils.distortion import dtw_workspace_bytes, launch_groups, mcd_batch
    pairs = [_case(1000 + i, Tr, Td, kind="int" if i % 3 == 0 else "rand") for i, (Tr, Td) in enumerate(SHAPES)]
    refs, decs = [p[0] for p in pairs], [p[1] for p in pairs]
    budget = 3 * dtw_workspace_bytes(300, 513)
    groups = launch_groups([len(a) for a in refs], [len(b) for b in decs], budget)
    assert len(groups) >= 4 and any(b - a > 1 for a, b, _ in groups)
    split = _check(pairs, True, workspace_bytes=budget)
    whole = mcd_batch(refs, decs, dtw=True, return_path=True)
    again = mcd_batch(refs, decs, dtw=True, return_path=True, workspace_bytes=budget)
    for r in (whole, again):
        assert np.array_equal(r.sums, split.sums) and np.array_equal(r.counts, split.counts)
        assert all(np.array_equal(p, q) for p, q in zip(r.paths, split.paths))
    no_path = mcd_batch(refs, decs, dtw=True)
    assert no_path.paths is None and np.array_equal(no_path.sums, split.sums)
    assert np.array_equal(no_path.counts, split.counts)
    aligned = mcd_batch(refs, decs)
    for k in (0, 5, 11, 16):
        alone = mcd_batch(refs[k:k + 1], decs[k:k + 1], dtw=True, return_path=True)
        assert np.array_equal(alone.sums[0], split.sums[k]) and np.array_equal(alone.paths[0], split.paths[k])
        one = mcd_batch(refs[k:k + 1], decs[k:k + 1])
        assert np.array_equal(one.sums[0], aligned.sums[k]) and one.counts[0] == aligned.counts[k]


def test_many_pairs_stride_over_the_grid():
    """More pairs than the DTW grid has CTAs: each CTA takes several pairs, each pair at its own workspace offset."""
    import torch
    from pytorchwavenetvocoder_b200.utils.distortion import mcd_batch
    n = 3 * torch.cuda.get_device_properties(0).multi_processor_count + 5
    rng = np.random.RandomState(9)
    lens = rng.randint(1, 40, size=(n, 2))
    pairs = [(_frames(rng, a, 25, "rand"), _frames(rng, b, 25, "int")) for a, b in lens]
    got = _check(pairs, True)
    assert np.array_equal(mcd_batch([p[0] for p in pairs], [p[1] for p in pairs], dtw=True).sums, got.sums)
    _check(pairs, False)


# ---- the CLI end to end ----------------------------------------------------------------------------------------------

def _speechlike(rng, n, amp=6000.0):
    from scipy.signal import lfilter
    e = rng.randn(n) * 300.0
    e[::97] += amp
    y = lfilter([1.0], [1.0, -1.4, 0.75, -0.15], e)
    return np.int16(y / (np.abs(y).max() + 1e-9) * amp)


def _run(args):
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.calc_mcd"] + args, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return r.returncode, r.stdout.decode()


def _tsv(path):
    rows = [line.rstrip("\n").split("\t") for line in open(path)][1:]
    return {r[0]: (int(r[1]), float(r[2])) for r in rows}


def test_cli_end_to_end(tmp_path):
    from scipy.io import wavfile
    from pytorchwavenetvocoder_b200.utils.distortion import corpus_mcd, mcd_wavs
    rng = np.random.RandomState(4)
    nat, same, noisy, slow = (tmp_path / d for d in ("nat", "same", "noisy", "slow"))
    for d in (nat, same, noisy, slow):
        d.mkdir()
    xs = {"a": _speechlike(rng, 16000), "b": _speechlike(rng, 24001)}
    ys, zs = {}, {}
    for k, x in xs.items():
        wavfile.write(str(nat / (k + ".wav")), 16000, x)
        wavfile.write(str(same / (k + ".wav")), 16000, x)
        ys[k] = np.int16(np.clip(x + rng.randn(len(x)) * 200, -32768, 32767))
        wavfile.write(str(noisy / (k + ".wav")), 16000, ys[k])
        zs[k] = x[np.minimum((np.arange(int(len(x) * 1.1)) / 1.1).astype(int), len(x) - 1)]
        wavfile.write(str(slow / (k + ".wav")), 16000, zs[k])

    out = str(tmp_path / "same.tsv")
    rc, log = _run(["--reference", str(nat), "--decoded", str(same), "--outfile", out])
    assert rc == 0, log
    t = _tsv(out)
    assert t["a"] == (188, 0.0) and t["b"][1] == 0.0 and t["<corpus>"][1] == 0.0

    out = str(tmp_path / "noisy.tsv")
    rc, log = _run(["--reference", str(nat), "--decoded", str(noisy), "--outfile", out, "--batch_size", "1"])
    assert rc == 0, log
    t = _tsv(out)
    want = mcd_wavs([xs["a"], xs["b"]], [ys["a"], ys["b"]], 16000, 1024, 80, 24, 0.41, highpass_cutoff=70)
    assert t["a"] == (want.counts[0], want.mcd[0]) and t["b"] == (want.counts[1], want.mcd[1])
    assert want.mcd.min() > 0 and t["<corpus>"] == (int(want.counts.sum()), corpus_mcd(want)[0])
    assert "corpus MCD" in log

    out = str(tmp_path / "slow.tsv")
    rc, log = _run(["--reference", str(nat), "--decoded", str(slow), "--outfile", out])
    assert rc == 1 and "--dtw" in log and str(slow / "a.wav") in log and not os.path.exists(out)
    rc, log = _run(["--reference", str(nat), "--decoded", str(slow), "--outfile", out, "--dtw"])
    assert rc == 0, log
    t = _tsv(out)
    want = mcd_wavs([xs["a"], xs["b"]], [zs["a"], zs["b"]], 16000, 1024, 80, 24, 0.41, highpass_cutoff=70, dtw=True)
    assert t["a"] == (want.counts[0], want.mcd[0]) and t["b"] == (want.counts[1], want.mcd[1])
    assert want.counts[0] >= 208 and np.all(np.isfinite(want.mcd)) and want.mcd.min() > 0
