# -*- coding: utf-8 -*-
"""CPU tier of the mcep features (DESIGN.md §6 row f6): wnb_mcep's argument checks, the host tables of utils/mcep.py
against numpy and the oracle, the recipes' stage 1 mcep argument lists, and the too-short-utterance error, up to the
point where the GPU would start."""
import logging
import os

import numpy as np
import pytest

from oracle import mcep_oracle as MO

WNB_ERR_INVALID, WNB_ERR_UNSUPPORTED = -1, -3


def _call(lib, fake=16, **kw):
    a = dict(x=fake, x_is_i16=1, offsets=fake, frame_offsets=fake, n_utts=1, n_frames=10, fftl=1024, hop=80, order=25,
             alpha=0.41, window=fake, twiddles=fake, warp_cos=fake, init_map=fake, neg_alpha_pow=fake, miniter=2,
             maxiter=30, threshold=1e-3, eps=1e-10, min_det=1e-6, out=fake, iters=fake, stream=None)
    a.update(kw)
    return lib.wnb_mcep(*a.values())


def test_wnb_mcep_argument_checks():
    from pytorchwavenetvocoder_b200._lib import load
    lib = load()
    for name in ("x", "offsets", "frame_offsets", "window", "twiddles", "warp_cos", "init_map", "neg_alpha_pow", "out",
                 "iters"):
        assert _call(lib, **{name: None}) == WNB_ERR_INVALID
        assert b"null pointer" in lib.wnb_last_error()
    for kw in (dict(n_utts=0), dict(n_frames=0), dict(hop=0), dict(maxiter=-1), dict(maxiter=1001), dict(eps=0.0),
               dict(threshold=-1.0)):
        assert _call(lib, **kw) == WNB_ERR_INVALID, kw
    for kw in (dict(fftl=512), dict(fftl=8192), dict(fftl=1000), dict(order=0), dict(order=41), dict(alpha=-0.01),
               dict(alpha=0.61), dict(alpha=float("nan"))):
        assert _call(lib, **kw) == WNB_ERR_UNSUPPORTED, kw
        assert b"not supported" in lib.wnb_last_error()


def test_warped_cos_against_numpy_phase():
    from pytorchwavenetvocoder_b200.utils.mcep import warped_cos
    for L, a in ((1024, 0.41), (1024, 0.455), (2048, 0.0), (4096, 0.6)):
        w = 2 * np.pi * np.arange(L // 2 + 1) / L
        th = w + 2 * np.arctan(a * np.sin(w) / (1 - a * np.cos(w)))
        assert np.abs(warped_cos(L, a) - np.cos(th)).max() < 4e-15   # numpy's own rounding


@pytest.mark.parametrize("L,M,a", [(1024, 25, 0.41), (1024, 35, 0.455), (2048, 24, 0.41), (1024, 40, 0.6)])
def test_init_map_is_the_oracle_initial_value(L, M, a):
    """W log P equals the oracle's FFT-and-freqt initial value (and its convergence seed) on a speech-like frame."""
    from pytorchwavenetvocoder_b200.utils.mcep import init_map
    rng = np.random.RandomState(L + M)
    x = np.cumsum(rng.randn(L)) * 100 + rng.randn(L) * 10
    frame = x * MO.hamming(L)
    P = np.abs(np.fft.rfft(frame)) ** 2 + 1e-10
    W = init_map(L, M, a)
    assert W.shape == (M + 2, L // 2 + 1) and W.dtype == np.float64
    mc, s = MO.initial_value(frame, M, a)
    got = W @ np.log(P)
    assert np.abs(got[:M + 1] - mc).max() < 1e-12 * (1 + np.abs(mc).max())
    assert abs(got[M + 1] - s) < 1e-12 * (1 + abs(s))


def test_neg_alpha_powers_and_window():
    from pytorchwavenetvocoder_b200.utils.mcep import hamming_window, n_frames, neg_alpha_powers
    al = neg_alpha_powers(35, 0.455)
    assert al[0] == 1.0 and np.allclose(al, (-0.455) ** np.arange(36), rtol=1e-14, atol=0)
    assert np.array_equal(hamming_window(1024), MO.hamming(1024))
    for n in (1023, 1024, 1025, 1103, 1104, 16000):
        assert n_frames(n, 1024, 80) == MO.n_frames(n, 1024, 80)


RECIPE_MCEP_ARGS = {
    "arctic": ["--waveforms", "data/tr/wav.scp", "--wavdir", "wav_hpf/tr", "--hdf5dir", "hdf5/tr", "--feature_type",
               "mcep", "--fs", "16000", "--shiftms", "5", "--mcep_dim", "25", "--mcep_alpha", "0.410",
               "--highpass_cutoff", "70", "--save_wav", "false", "--fftl", "1024", "--n_jobs", "10"],
    "ljspeech": ["--waveforms", "data/tr/wav.scp", "--wavdir", "wav_hpf/tr", "--hdf5dir", "hdf5/tr", "--feature_type",
                 "mcep", "--fs", "22050", "--shiftms", "11.61", "--mcep_dim", "35", "--mcep_alpha", "0.455",
                 "--highpass_cutoff", "70", "--save_wav", "false", "--fftl", "1024", "--n_jobs", "10"],
}


@pytest.mark.parametrize("recipe", sorted(RECIPE_MCEP_ARGS))
def test_recipe_stage1_mcep_arguments_parse(recipe):
    from pytorchwavenetvocoder_b200.bin.feature_extract import get_parser
    from pytorchwavenetvocoder_b200.utils.melspc import shift_length
    a = get_parser().parse_args(RECIPE_MCEP_ARGS[recipe])
    assert a.feature_type == "mcep" and a.save_wav == 0 and a.fftl == 1024 and a.highpass_cutoff == 70
    assert (a.mcep_dim, a.mcep_alpha, shift_length(a.shiftms, a.fs)) == \
        ((25, 0.41, 80) if recipe == "arctic" else (35, 0.455, 256))
    assert get_parser().parse_args(["--feature_type", "mcep"]).mcep_dim == 24


def test_too_short_utterance_is_an_error():
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    with pytest.raises(ValueError, match="utterance 1 has 1023 samples, fewer than fftl = 1024"):
        mcep_batch([np.zeros(2000, np.int16), np.zeros(1023, np.int16)], 16000, 1024, 80, 25, 0.41)


def test_cli_too_short_wav_exits_1_naming_the_file(tmp_path, caplog):
    from scipy.io import wavfile
    from pytorchwavenetvocoder_b200.bin import feature_extract as fe
    os.makedirs(str(tmp_path / "wav"))
    wavfile.write(str(tmp_path / "wav" / "short.wav"), 16000, np.zeros(1000, dtype=np.int16))
    with caplog.at_level(logging.ERROR), pytest.raises(SystemExit) as e:
        fe.main(["--waveforms", str(tmp_path / "wav"), "--hdf5dir", str(tmp_path / "h5"), "--wavdir",
                 str(tmp_path / "hpf"), "--feature_type", "mcep", "--save_wav", "false", "--verbose", "0"])
    assert e.value.code == 1 and "short.wav has 1000 samples" in caplog.text
    assert not os.path.exists(str(tmp_path / "h5"))       # checked before anything is written


def test_cli_checks_every_length_before_writing(tmp_path, caplog):
    from scipy.io import wavfile
    from pytorchwavenetvocoder_b200.bin import feature_extract as fe
    os.makedirs(str(tmp_path / "wav"))
    for name, n in (("a.wav", 5000), ("b.wav", 1023), ("c.wav", 1024), ("d.wav", 10)):
        wavfile.write(str(tmp_path / "wav" / name), 16000, np.zeros(n, dtype=np.int16))
    with caplog.at_level(logging.ERROR), pytest.raises(SystemExit) as e:
        fe.main(["--waveforms", str(tmp_path / "wav"), "--hdf5dir", str(tmp_path / "h5"), "--wavdir",
                 str(tmp_path / "hpf"), "--feature_type", "mcep", "--verbose", "0"])
    assert e.value.code == 1
    assert "b.wav has 1023 samples" in caplog.text and "d.wav has 10 samples" in caplog.text
    assert "a.wav" not in caplog.text and "c.wav" not in caplog.text
    assert not os.path.exists(str(tmp_path / "h5")) and not os.path.exists(str(tmp_path / "hpf"))


def test_cli_world_still_exits_1(tmp_path, caplog):
    from pytorchwavenetvocoder_b200.bin import feature_extract as fe
    with caplog.at_level(logging.ERROR), pytest.raises(SystemExit) as e:
        fe.main(["--waveforms", str(tmp_path), "--hdf5dir", str(tmp_path / "h5"), "--feature_type", "world",
                 "--verbose", "0"])
    assert e.value.code == 1 and "WORLD" in caplog.text and not os.path.exists(str(tmp_path / "h5"))

