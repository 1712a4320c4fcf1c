# -*- coding: utf-8 -*-
"""GPU tier: wnb_mlsa_filter (csrc/mlsa.cu, SURVEY.md 8 row f4) against the CPU oracle (oracle/mlsa_oracle.c) -- bit exact
in float64 and through the int16 wav path, ragged batches, both Pade orders, the inverse filter, a full-length batch
(64 x 160 000 samples) checked exactly on a subset and through the shaping -> restoring round trip, and the CLI mirror
of reference bin/noise_shaping.py end to end."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _coef(rng, order, mag, alpha):
    from oracle import mlsa_oracle as M
    return M.convert_mcep_to_mlsa_coef(rng.randn(order + 1) * 0.6, mag, alpha)


def _speechlike(rng, n, amp=3000.0):
    x = np.cumsum(rng.randn(n))
    x -= np.linspace(x[0], x[-1], n)
    return x / (np.abs(x).max() + 1e-9) * amp + rng.randn(n) * 20.0


@pytest.mark.parametrize("order,alpha,pd", [(24, 0.41, 4), (24, 0.41, 5), (59, 0.455, 4), (2, 0.35, 4)])
def test_ragged_batch_float64_bit_exact(order, alpha, pd):
    from oracle import mlsa_oracle as M
    from pytorchwavenetvocoder_b200.utils.mlsa import mlsa_filter_batch
    rng = np.random.RandomState(order * 10 + pd)
    coef = _coef(rng, order, 0.5, alpha)
    lens = [0, 1, 7, 8, 9, 1000, 3001, 15, 64]           # 9 utterances: three warps, the last one partly empty
    xs = [_speechlike(rng, n) if n > 1 else rng.randn(n) * 100 for n in lens]
    for c in (coef, -coef):                              # noise shaping and its inverse (reference noise_shaping.py:55-56)
        got = mlsa_filter_batch(xs, c, alpha, pd=pd)
        for x, y in zip(xs, got):
            want = M.filter_const(x, c, alpha, pd)
            assert y.dtype == np.float64 and y.shape == want.shape
            assert np.array_equal(y, want), "max abs diff %g" % (np.abs(y - want).max() if len(y) else 0.0)


def test_int16_wav_path_bit_exact():
    from oracle import mlsa_oracle as M
    from pytorchwavenetvocoder_b200.utils.mlsa import mlsa_filter_batch
    rng = np.random.RandomState(5)
    coef = _coef(rng, 24, 0.5, 0.41)
    xs = [np.int16(_speechlike(rng, n, 12000.0)) for n in (4000, 2500, 801, 16000, 3)]
    got = mlsa_filter_batch(xs, coef, 0.41)
    for x, y in zip(xs, got):
        assert y.dtype == np.int16
        assert np.array_equal(y, M.noise_shaping_one(x, coef, 0.41))
    # float64 out of int16 in (np.float64(x) conversion inside the kernel)
    gotf = mlsa_filter_batch(xs, coef, 0.41, out_int16=False)
    for x, y in zip(xs, gotf):
        assert np.array_equal(y, M.filter_const(np.float64(x), coef, 0.41))


def test_full_length_batch_exact_subset_and_round_trip():
    """configs[3]'s decode output size: 64 utterances x 160 000 samples.  Three of them are compared with the oracle bit
    for bit; all of them must come back through the inverse filter (shaping -> restoring, recipes' stage 3 / stage 6)."""
    from oracle import mlsa_oracle as M
    from pytorchwavenetvocoder_b200.utils.mlsa import mlsa_filter_batch
    rng = np.random.RandomState(6)
    coef = _coef(rng, 24, 0.5, 0.41)
    n = 160000
    xs = [_speechlike(rng, n - (i % 5) * 37) for i in range(64)]
    ys = mlsa_filter_batch(xs, coef, 0.41)
    for i in (0, 31, 63):
        assert np.array_equal(ys[i], M.filter_const(xs[i], coef, 0.41))
    back = mlsa_filter_batch(ys, -coef, 0.41)
    worst = max(np.abs(b - x).max() / np.abs(x).max() for b, x in zip(back, xs))
    print("round trip through the inverse filter: worst relative error %.2e" % worst)
    assert worst < 1e-3
    assert all(len(y) == len(x) for x, y in zip(xs, ys))


def test_rejects_bad_arguments():
    import torch
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    off = torch.tensor([0, 8], dtype=torch.int64, device="cuda")
    b = torch.zeros(25, dtype=torch.float64, device="cuda")
    assert lib.wnb_mlsa_filter(_lib.ptr(x), 0, _lib.ptr(off), 1, _lib.ptr(b), 24, 0.41, 3, 1.0, _lib.ptr(x), 0, None) != 0
    assert b"pd must be 4 or 5" in lib.wnb_last_error()
    assert lib.wnb_mlsa_filter(_lib.ptr(x), 0, _lib.ptr(off), 1, _lib.ptr(b), 24, 1.5, 4, 1.0, _lib.ptr(x), 0, None) != 0


def test_cli_noise_shaping_and_restore(tmp_path):
    """reference bin/noise_shaping.py end to end: stats world/mean -> /mlsa/coef + /mlsa/alpha written, wav files shaped,
    then `--inv true` restores them (recipes' stage 3 and stage 6); int16 files equal the oracle's."""
    from scipy.io import wavfile
    from oracle import mlsa_oracle as M
    from pytorchwavenetvocoder_b200.bin import noise_shaping as ns
    from pytorchwavenetvocoder_b200.utils import read_hdf5, write_hdf5
    rng = np.random.RandomState(7)
    wavdir, outdir, invdir = tmp_path / "wav", tmp_path / "ns", tmp_path / "restored"
    wavdir.mkdir()
    xs = {}
    for i, n in enumerate((8000, 12345, 4001)):
        xs["u%d.wav" % i] = np.int16(_speechlike(rng, n, 9000.0))
        wavfile.write(str(wavdir / ("u%d.wav" % i)), 16000, xs["u%d.wav" % i])
    stats = str(tmp_path / "stats.npz")
    mean = rng.randn(28) * 0.5                            # world features: [uv, f0, mcep 0..24, ap] -> mcep = mean[2:27]
    write_hdf5(stats, "/world/mean", mean)
    ns.main(["--waveforms", str(wavdir), "--stats", stats, "--outdir", str(outdir), "--fs", "16000", "--mag", "0.5",
             "--mcep_alpha", "0.41", "--batch_size", "2", "--verbose", "0"])
    coef = M.convert_mcep_to_mlsa_coef(mean[2:27], 0.5, 0.41)
    assert np.array_equal(read_hdf5(stats, "/mlsa/coef"), coef) and float(read_hdf5(stats, "/mlsa/alpha")) == 0.41
    for name, x in xs.items():
        fs, y = wavfile.read(str(outdir / name))
        assert fs == 16000 and y.dtype == np.int16 and np.array_equal(y, M.noise_shaping_one(x, coef, 0.41))
    ns.main(["--waveforms", str(outdir), "--stats", stats, "--outdir", str(invdir), "--fs", "16000", "--inv", "true",
             "--verbose", "0"])
    for name, x in xs.items():
        _, shaped = wavfile.read(str(outdir / name))
        _, r = wavfile.read(str(invdir / name))
        assert np.array_equal(r, M.noise_shaping_one(shaped, -coef, 0.41))
        assert np.abs(np.float64(r) - np.float64(x)).max() < 0.002 * np.abs(np.float64(x)).max() + 4    # int16 truncation twice
