# -*- coding: utf-8 -*-
"""CPU tier of the melspc features (DESIGN.md §6 row f5): the float64 restatement in tests/melspc_reference.py pinned by
what its pieces are, the host tables of utils/melspc.py against it bit for bit, the closed-form reflect map, the int16
cast rule, the library's argument checks, and the two CLIs (bin/feature_extract.py, bin/calc_stats.py) up to the point
where the GPU would start."""
import logging
import os
import warnings

import numpy as np
import pytest

from tests import melspc_reference as R


def test_slaney_mel_scale_documented_values():
    assert R.slaney_hz_to_mel(60.0) == pytest.approx(0.9, rel=1e-15)
    assert R.slaney_mel_to_hz(3.0) == pytest.approx(200.0, rel=1e-15)
    assert R.slaney_hz_to_mel(1000.0) == pytest.approx(15.0, rel=1e-15)
    f = np.array([0.0, 300.0, 999.0, 1000.0, 2500.0, 8000.0, 11025.0])
    assert np.allclose(R.slaney_mel_to_hz(R.slaney_hz_to_mel(f)), f, rtol=1e-13, atol=1e-12)
    from pytorchwavenetvocoder_b200.utils import melspc as M
    assert M.hz_to_mel(60) == R.slaney_hz_to_mel(60.0) and M.mel_to_hz(3) == R.slaney_mel_to_hz(3.0)
    assert np.array_equal(M.hz_to_mel(f), R.slaney_hz_to_mel(f))


@pytest.mark.parametrize("fs,fftl,n_mels,fmin,fmax", [(16000, 1024, 80, 0, 8000), (22050, 1024, 80, 0, 11025),
                                                      (16000, 1024, 80, 80, 7600), (22050, 2048, 40, 125, 7600)])
def test_filter_peaks_and_unit_area(fs, fftl, n_mels, fmin, fmax):
    """Each filter peaks at one of the two bins around its centre frequency (the middle of its three mel points; the
    triangle is asymmetric in Hz above 1 kHz, so not always the nearer one), and a filter
    several bins wide integrates to 1 over Hz (Slaney area normalisation); the Riemann sum of a triangle sampled every
    df Hz is within 6 df / width of its integral."""
    basis = R.mel_basis(fs, fftl, n_mels, fmin, fmax).astype(np.float64)
    df = fs / fftl
    edges = R.slaney_mel_to_hz(np.linspace(R.slaney_hz_to_mel(float(fmin)), R.slaney_hz_to_mel(float(fmax)), n_mels + 2))
    bins = np.arange(fftl // 2 + 1) * df
    wide = 0
    for i in range(n_mels):
        if not basis[i].any():
            continue
        peak = bins[np.argmax(basis[i])]
        assert abs(peak - edges[i + 1]) < df, (i, peak, edges[i + 1])
        width = edges[i + 2] - edges[i]
        if width >= 10 * df:
            wide += 1
            assert abs(basis[i].sum() * df - 1.0) <= 6 * df / width + 1e-6, (i, basis[i].sum() * df)
    assert wide >= n_mels // 4


@pytest.mark.parametrize("fs,fftl,n_mels,fmin,fmax", [(16000, 1024, 80, None, None), (22050, 1024, 80, None, None),
                                                      (16000, 1024, 80, 80, 7600), (22050, 1024, 40, 125, 7600),
                                                      (16000, 64, 40, None, None), (24000, 4096, 80, None, None)])
def test_product_filterbank_equals_oracle_bit_for_bit(fs, fftl, n_mels, fmin, fmax):
    from pytorchwavenetvocoder_b200.utils.melspc import mel_filterbank
    fmin_ = 0 if fmin is None else fmin
    fmax_ = fs // 2 if fmax is None else fmax
    table, lo, hi = mel_filterbank(fs, fftl, n_mels, fmin_, fmax_)
    want = R.mel_basis(fs, fftl, n_mels, fmin_, fmax_)
    assert table.dtype == np.float32 and table.shape == (n_mels, fftl // 2 + 1)
    assert np.array_equal(table.view(np.uint32), want.view(np.uint32))
    for i in range(n_mels):           # [lo, hi) holds exactly the nonzero bins, which are contiguous
        nz = np.flatnonzero(table[i])
        assert np.array_equal(nz, np.arange(lo[i], hi[i])), i


def test_hop_arithmetic():
    from pytorchwavenetvocoder_b200.utils.melspc import n_frames, shift_length
    assert shift_length(5, 16000) == 80
    assert shift_length(11.61, 22050) == 256
    assert shift_length(16, 16000) == 256
    assert n_frames(160000, 80) == 2001 and n_frames(1, 80) == 1 and n_frames(80, 80) == 2


@pytest.mark.parametrize("fftl", [64, 256])
def test_reflect_map_equals_numpy_pad(fftl):
    from pytorchwavenetvocoder_b200.utils.melspc import reflect_index
    pad = fftl // 2
    for n in range(1, fftl + 2):
        x = np.arange(n)
        want = np.pad(x, pad, mode="reflect")
        got = x[reflect_index(np.arange(-pad, n + pad), n)]
        assert np.array_equal(got, want), n


@pytest.mark.parametrize("fftl", [64, 1024])
def test_oracle_stft_bin_centred_cosine_and_parseval(fftl):
    """A cosine of amplitude A at bin k0 over a whole frame gives |X[k0]| = A fftl / 4 under the periodic Hann window
    (its DFT is fftl/2 at bin 0 and -fftl/4 at bins +-1); Parseval holds per frame."""
    rng = np.random.RandomState(fftl)
    hop = fftl // 4
    A = 0.3
    for k0 in (2, 5, fftl // 4 + 1, fftl // 2 - 2):
        n = np.arange(8 * fftl)
        x = 32768 * A * np.cos(2 * np.pi * k0 * n / fftl + rng.uniform(0, 2 * np.pi))
        S = R.magnitude(x, fftl, hop)
        for t in (3, 10, 20):          # frames fully inside the signal
            assert S[t, k0] == pytest.approx(A * fftl / 4, rel=1e-12)
    x = rng.randn(3000) * 5000
    fr = R.frames(x / 32768, fftl, hop) * R.hann(fftl)
    S = R.magnitude(x, fftl, hop)
    energy = S[:, 0] ** 2 + S[:, -1] ** 2 + 2 * (S[:, 1:-1] ** 2).sum(axis=1)
    assert np.allclose(energy, fftl * (fr ** 2).sum(axis=1), rtol=1e-12)


def test_hann_window_is_periodic():
    for fftl in (64, 1024):
        n = np.arange(fftl)
        assert np.allclose(R.hann(fftl), 0.5 - 0.5 * np.cos(2 * np.pi * n / fftl), atol=1e-15, rtol=0)


def test_oracle_fir_equals_scipy_lfilter():
    from scipy.signal import lfilter
    from pytorchwavenetvocoder_b200.utils.melspc import lowcut_taps
    rng = np.random.RandomState(1)
    for fs, cutoff, n in ((16000, 70, 5000), (22050, 70, 300), (16000, 300, 100)):
        taps = lowcut_taps(fs, cutoff)
        x = np.float64(np.int16(rng.randn(n) * 8000))
        y, mag = R.lowcut(x, taps)
        want = lfilter(taps, 1, x)
        assert np.all(np.abs(y - want) <= R.fir_bound(mag)), np.abs(y - want).max()
    taps = lowcut_taps(16000, 70)       # sum |b| = 1.87: a full-scale input can overshoot int16, which the cast wraps
    assert len(taps) == 255 and abs(np.abs(taps).sum() - 1.87) < 0.01


def test_int16_cast_rule_matches_numpy():
    from pytorchwavenetvocoder_b200.utils.melspc import int16_cast
    v = np.array([40000.7, 3e9, -3e9, 65535.9, -40000.2, 32767.99, -32768.5, -32769.0, 1e20, -1e20, 2147483647.5,
                  -2147483648.7, -2147483649.0, 2147483648.0, 0.5, -0.5, -1.9, 61000.0, -61000.0, np.nan])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.int16(v)
    assert np.array_equal(int16_cast(v), want), (int16_cast(v), want)
    assert int16_cast(np.array([40000.7]))[0] == -25536 and int16_cast(np.array([3e9]))[0] == 0


def test_library_rejects_bad_arguments_without_gpu():
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    p = 4096          # any non-null value: the checks run before any device work
    assert lib.wnb_melspc(p, 0, p, p, 1, 1, 1000, 80, p, p, p, p, p, 80, p, None) == -3
    assert b"fftl 1000" in lib.wnb_last_error()
    assert lib.wnb_melspc(p, 0, p, p, 1, 1, 8192, 80, p, p, p, p, p, 80, p, None) == -3
    assert lib.wnb_melspc(p, 0, p, p, 1, 1, 32, 80, p, p, p, p, p, 80, p, None) == -3
    assert lib.wnb_melspc(p, 0, p, p, 2, 1, 1024, 80, p, p, p, p, p, 80, p, None) == -1      # fewer frames than utterances
    assert lib.wnb_melspc(None, 0, p, p, 1, 1, 1024, 80, p, p, p, p, p, 80, p, None) == -1
    assert lib.wnb_melspc(p, 0, p, p, 1, 1, 1024, 0, p, p, p, p, p, 80, p, None) == -1
    assert lib.wnb_melspc_lowcut(p, 1, p, 1, 100, p, 0, p, None, None) == -1
    assert lib.wnb_melspc_lowcut(p, 1, p, 1, 100, p, 1025, p, None, None) == -1
    assert lib.wnb_melspc_lowcut(p, 1, p, 0, 100, p, 255, p, None, None) == -1
    assert lib.wnb_melspc_lowcut(None, 1, p, 1, 100, p, 255, p, None, None) == -1


# ---- CLIs ------------------------------------------------------------------------------------------------------------
RECIPE_ARGS = {   # egs/*/sd-melspc/run.sh stage 1, with the recipes' empty fmin / fmax
    "arctic": ["--waveforms", "data/tr/wav.scp", "--wavdir", "wav_hpf/tr", "--hdf5dir", "hdf5/tr", "--feature_type",
               "melspc", "--fs", "16000", "--shiftms", "5", "--mspc_dim", "80", "--highpass_cutoff", "70", "--fftl",
               "1024", "--fmin", "", "--fmax", "", "--n_jobs", "10"],
    "ljspeech": ["--waveforms", "data/tr/wav.scp", "--wavdir", "wav_hpf/tr", "--hdf5dir", "hdf5/tr", "--feature_type",
                 "melspc", "--fs", "22050", "--shiftms", "11.61", "--mspc_dim", "80", "--highpass_cutoff", "70",
                 "--fftl", "1024", "--fmin", "", "--fmax", "", "--n_jobs", "10"],
}


@pytest.mark.parametrize("recipe", sorted(RECIPE_ARGS))
def test_feature_extract_parses_recipe_arguments(recipe):
    from pytorchwavenetvocoder_b200.bin.feature_extract import get_parser
    a = get_parser().parse_args(RECIPE_ARGS[recipe])
    assert a.feature_type == "melspc" and a.fmin is None and a.fmax is None and a.save_wav == 1 and a.fftl == 1024
    a = get_parser().parse_args(RECIPE_ARGS[recipe][:-6] + ["--fmin", "80", "--fmax", "7600", "--save_wav", "false"])
    assert a.fmin == 80 and a.fmax == 7600 and a.save_wav == 0
    a = get_parser().parse_args(["--feature_type", "mcep", "--mcep_dim", "25", "--mcep_alpha", "0.410", "--minf0", "60",
                                 "--maxf0", "300", "--fmin", "--batch_size", "8"])
    assert a.mcep_dim == 25 and a.fmin is None and a.batch_size == 8


def _write_wavs(d, fs, lens, seed=0):
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    os.makedirs(d, exist_ok=True)
    names = []
    for i, n in enumerate(lens):
        p = os.path.join(d, "u%d.wav" % i)
        wavfile.write(p, fs, np.int16(rng.randn(n) * 3000))
        names.append(p)
    return names


@pytest.mark.parametrize("ftype,needs", [("world", "WORLD"), ("mcep", "pysptk")])
def test_feature_extract_rejects_world_and_mcep(tmp_path, caplog, ftype, needs):
    from pytorchwavenetvocoder_b200.bin import feature_extract as fe
    _write_wavs(str(tmp_path / "wav"), 16000, [400])
    with caplog.at_level(logging.ERROR), pytest.raises(SystemExit) as e:
        fe.main(["--waveforms", str(tmp_path / "wav"), "--hdf5dir", str(tmp_path / "h5"), "--wavdir",
                 str(tmp_path / "hpf"), "--feature_type", ftype, "--verbose", "0"])
    assert e.value.code == 1
    assert "feature_extract.py" in caplog.text and needs in caplog.text
    assert not os.path.exists(str(tmp_path / "h5"))


def test_feature_extract_sampling_rate_mismatch_exits_1(tmp_path):
    from pytorchwavenetvocoder_b200.bin import feature_extract as fe
    _write_wavs(str(tmp_path / "wav"), 22050, [400, 500])
    with pytest.raises(SystemExit) as e:
        fe.main(["--waveforms", str(tmp_path / "wav"), "--hdf5dir", str(tmp_path / "h5"), "--wavdir",
                 str(tmp_path / "hpf"), "--feature_type", "melspc", "--fs", "16000", "--verbose", "0"])
    assert e.value.code == 1


def test_calc_stats_equals_sklearn_through_npz(tmp_path):
    from sklearn.preprocessing import StandardScaler
    from pytorchwavenetvocoder_b200.bin import calc_stats as cs
    from pytorchwavenetvocoder_b200.utils import read_hdf5, write_hdf5
    rng = np.random.RandomState(3)
    for ftype, dim in (("world", 28), ("melspc", 80), ("mcep", 25)):
        files, feats = [], []
        for i in range(5):
            f = (rng.randn(rng.randint(30, 200), dim) * rng.uniform(0.5, 3, dim) + rng.randn(dim)).astype(np.float32)
            p = str(tmp_path / ("%s_%d.npz" % (ftype, i)))
            write_hdf5(p, "/" + ftype, f)
            files.append(p)
            feats.append(f)
        lst = str(tmp_path / ("%s.scp" % ftype))
        open(lst, "w").write("\n".join(files) + "\n")
        stats = str(tmp_path / "stats.npz")
        cs.main(["--feats", lst, "--stats", stats, "--feature_type", ftype, "--verbose", "0"])
        sc = StandardScaler()
        for f in feats:
            sc.partial_fit(f)
        mean, scale = sc.mean_.copy(), sc.scale_.copy()
        if ftype == "world":
            mean[0], scale[0] = 0.0, 1.0
        got_m, got_s = read_hdf5(stats, "/%s/mean" % ftype), read_hdf5(stats, "/%s/scale" % ftype)
        assert got_m.dtype == np.float32 and got_s.dtype == np.float32
        assert np.array_equal(got_m, np.float32(mean)) and np.array_equal(got_s, np.float32(scale))
    assert read_hdf5(stats, "/world/mean").shape == (28,) and read_hdf5(stats, "/melspc/scale").shape == (80,)


def test_noise_shaping_uses_the_shared_wav_helpers():
    from pytorchwavenetvocoder_b200.bin import noise_shaping as ns
    from pytorchwavenetvocoder_b200 import utils
    assert ns.read_wav_int16 is utils.read_wav_int16 and ns.write_wav_int16 is utils.write_wav_int16
