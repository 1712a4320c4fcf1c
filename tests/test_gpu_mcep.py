# -*- coding: utf-8 -*-
"""GPU tier: STFT mel-cepstra (wnb_mcep, utils/mcep.py mcep_batch, bin/feature_extract.py --feature_type mcep) frame by
frame against oracle/mcep_oracle.c, and the sd-melspc recipe's noise-shaping stages end to end through the CLIs.  The
bar and the checker are in tests/mcep_check.py; the corners of the supported range and every exit of the Newton loop
are in tests/test_gpu_mcep_edges.py."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mcep_oracle as MO
from tests.mcep_check import _check, _speechlike

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARCTIC = dict(fs=16000, fftl=1024, hop=80, order=25, alpha=0.41)
LJSPEECH = dict(fs=22050, fftl=1024, hop=256, order=35, alpha=0.455)
CLI_DEFAULT = dict(fs=16000, fftl=1024, hop=80, order=24, alpha=0.41)


@pytest.mark.parametrize("cfg,name", [(ARCTIC, "arctic"), (LJSPEECH, "ljspeech"), (CLI_DEFAULT, "cli-default")])
@pytest.mark.parametrize("cutoff", [70, 0])
@pytest.mark.parametrize("as_int16", [True, False])
def test_ragged_against_oracle(cfg, name, cutoff, as_int16):
    seed = {"arctic": 1, "ljspeech": 2, "cli-default": 3}[name] * 4 + (cutoff == 70) * 2 + as_int16
    rng = np.random.RandomState(seed)
    L, hop = cfg["fftl"], cfg["hop"]
    lens = [L, L + 1, L + hop - 1, L + hop, 16000, 160000]
    xs = [_speechlike(rng, n) for n in lens]
    xs = [np.int16(x) for x in xs] if as_int16 else [np.float64(np.int16(x)) + rng.uniform(-0.5, 0.5, len(x))
                                                      for x in xs]
    which = range(len(xs)) if cutoff == 70 and as_int16 else range(len(xs) - 1)
    _check(xs, cfg["fs"], L, hop, cfg["order"], cfg["alpha"], cutoff, which=which,
           label="%s cutoff %d %s" % (name, cutoff, "int16" if as_int16 else "float64"))


def test_fftl_2048():
    rng = np.random.RandomState(11)
    xs = [np.int16(_speechlike(rng, n)) for n in (2048, 2049, 9000)]
    _check(xs, 16000, 2048, 80, 25, 0.41, 70, label="fftl 2048")
    _check(xs, 16000, 2048, 160, 40, 0.6, 0, label="fftl 2048 order 40 alpha 0.6")


def test_exact_model_recovery_on_gpu():
    """a one-frame signal whose Hamming-windowed frame carries exp(2 sum c*_m cos(m w~_k)) as its periodogram plus eps"""
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    for M, a in ((24, 0.41), (35, 0.455), (25, 0.0)):
        rng = np.random.RandomState(M)
        cs = rng.randn(M + 1) * 0.6 / np.arange(1, M + 2)
        cs[0] = 4.0
        w = 2 * np.pi * np.arange(1024) / 1024
        th = np.arctan2((1 - a * a) * np.sin(w), (1 + a * a) * np.cos(w) - 2 * a)
        P = np.exp(2.0 * np.cos(np.outer(th, np.arange(M + 1))) @ cs) - 1e-10
        frame = np.fft.irfft(np.sqrt(P[:513]), 1024)
        x = frame / MO.hamming(1024)
        got = mcep_batch([x], 16000, 1024, 80, M, a, threshold=1e-14, maxiter=100)[0]
        assert got.shape == (1, M + 1)
        err = np.abs(got[0] - cs)
        assert np.all(err <= 1e-8 + np.spacing(np.abs(np.float32(cs)))), (M, a, err.max())


def test_digital_silence():
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    got = mcep_batch([np.zeros(3000, dtype=np.int16)], 16000, 1024, 80, 25, 0.41)[0]
    c0 = 0.5 * np.log(1e-10)
    assert np.all((got[:, 0] == np.float32(c0)) | (np.abs(got[:, 0] - c0) <= np.spacing(np.float32(c0))))
    assert np.abs(got[:, 1:]).max() < 1e-12


def test_full_scale_square_waves():
    xs = [np.int16(np.where((np.arange(n) // p) % 2 == 0, 32767, -32768)) for n, p in ((5000, 37), (4000, 100))]
    _check(xs, 16000, 1024, 80, 25, 0.41, 0, label="square int16")
    _check(xs, 16000, 1024, 80, 25, 0.41, 70, label="square lowcut")


def test_unsupported_shapes_raise():
    from pytorchwavenetvocoder_b200._lib import WnbError
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    x = [np.zeros(10000, dtype=np.int16)]
    for fftl, order, alpha in ((512, 25, 0.41), (8192, 25, 0.41), (1000, 25, 0.41), (1024, 41, 0.41),
                               (1024, 0, 0.41), (1024, 25, 0.7), (1024, 25, -0.1)):
        with pytest.raises(WnbError, match="not supported"):
            mcep_batch(x, 16000, fftl, 80, order, alpha)


def test_too_short_utterance_raises():
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    with pytest.raises(ValueError, match="utterance 1 has 1023 samples"):
        mcep_batch([np.zeros(2000, np.int16), np.zeros(1023, np.int16)], 16000, 1024, 80, 25, 0.41)


def test_two_runs_bit_identical():
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    rng = np.random.RandomState(4)
    xs = [np.int16(_speechlike(rng, n)) for n in (20000, 7001, 1024)]
    a, ia = mcep_batch(xs, 16000, 1024, 80, 25, 0.41, highpass_cutoff=70, return_iters=True)
    b, ib = mcep_batch(xs, 16000, 1024, 80, 25, 0.41, highpass_cutoff=70, return_iters=True)
    for u in range(3):
        assert np.array_equal(a[u].view(np.uint32), b[u].view(np.uint32)) and np.array_equal(ia[u], ib[u])


def test_full_size_batch():
    """64 x 160 000 samples at the arctic settings: every frame of three utterances and every 37th frame of the others"""
    rng = np.random.RandomState(8)
    xs = [np.int16(_speechlike(rng, 160000)) for _ in range(64)]
    _check(xs, 16000, 1024, 80, 25, 0.41, 70, which=(0, 31, 63), label="64 x 160000 full")
    _check(xs, 16000, 1024, 80, 25, 0.41, 70, which=range(1, 63, 5), stride=37, label="64 x 160000 strided")


def _run(args, timeout=600):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout)
    assert r.returncode == 0, r.stdout.decode()[-3000:]
    return r.stdout.decode()


def test_sd_melspc_noise_shaping_stages_end_to_end(tmp_path):
    """egs/arctic/sd-melspc stages 1, 2, 3 and 6 with its flags (stages 4 and 5 are in test_gpu_melspc.py)."""
    from scipy.io import wavfile
    from oracle import mlsa_oracle as MLSA
    from pytorchwavenetvocoder_b200.utils import read_hdf5
    from pytorchwavenetvocoder_b200.utils.mcep import mcep_batch
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    rng = np.random.RandomState(12)
    wavdir, hpf, h5 = tmp_path / "wav", tmp_path / "wav_hpf", tmp_path / "hdf5"
    wavdir.mkdir()
    names = ["u%d" % i for i in range(3)]
    xs = [np.int16(_speechlike(rng, n, 9000.0)) for n in (16000, 12345, 20000)]
    for k, x in zip(names, xs):
        wavfile.write(str(wavdir / (k + ".wav")), 16000, x)
    scp = tmp_path / "wav.scp"
    scp.write_text("".join(str(wavdir / (k + ".wav")) + "\n" for k in names))
    fe = ["-m", "pytorchwavenetvocoder_b200.bin.feature_extract", "--waveforms", str(scp), "--wavdir", str(hpf),
          "--hdf5dir", str(h5), "--fs", "16000", "--shiftms", "5"]
    # stage 1: melspc, then the mcep pass into the same feature files
    _run(fe + ["--feature_type", "melspc", "--mspc_dim", "80", "--highpass_cutoff", "70", "--fftl", "1024", "--fmin",
               "", "--fmax", "", "--n_jobs", "10", "--batch_size", "2"])
    _run(fe + ["--feature_type", "mcep", "--mcep_dim", "25", "--mcep_alpha", "0.410", "--highpass_cutoff", "70",
               "--save_wav", "false", "--fftl", "1024", "--n_jobs", "10", "--batch_size", "2"])
    mspc = melspc_batch(xs, 16000, 1024, 80, 80, highpass_cutoff=70)
    mcep = mcep_batch(xs, 16000, 1024, 80, 25, 0.41, highpass_cutoff=70)
    files = []
    for k, m, c in zip(names, mspc, mcep):
        ff = (glob.glob(str(h5 / (k + ".h5"))) + glob.glob(str(h5 / (k + ".npz"))))[0]
        files.append(ff)
        assert np.array_equal(read_hdf5(ff, "/melspc"), m)
        assert np.array_equal(read_hdf5(ff, "/mcep"), c)
    # stage 2: statistics of both feature types into one file
    fl = tmp_path / "feats.scp"
    fl.write_text("".join(f + "\n" for f in files))
    stats = str(tmp_path / "stats.npz")
    for ft in ("melspc", "mcep"):
        _run(["-m", "pytorchwavenetvocoder_b200.bin.calc_stats", "--feats", str(fl), "--stats", stats,
              "--feature_type", ft])
    allc = np.concatenate(mcep).astype(np.float64)
    assert read_hdf5(stats, "/melspc/mean").shape == (80,)
    mean = read_hdf5(stats, "/mcep/mean")
    assert mean.shape == (26,) and np.allclose(mean, allc.mean(axis=0), rtol=1e-5, atol=1e-5)
    # stage 3: noise weighting of the high-passed training wavs (the inverse filter)
    wl = tmp_path / "wav_hpf.scp"
    wl.write_text("".join(str(hpf / (k + ".wav")) + "\n" for k in names))
    _run(["-m", "pytorchwavenetvocoder_b200.bin.noise_shaping", "--waveforms", str(wl), "--stats", stats, "--outdir",
          str(tmp_path / "wav_nwf"), "--feature_type", "mcep", "--fs", "16000", "--shiftms", "5", "--mcep_alpha",
          "0.410", "--mag", "0.5", "--inv", "true", "--n_jobs", "10"])
    coef = np.array(read_hdf5(stats, "/mlsa/coef"), dtype=np.float64)
    assert np.array_equal(coef, MLSA.convert_mcep_to_mlsa_coef(np.array(mean, dtype=np.float64), 0.5, 0.41))
    for k in names:
        _, x = wavfile.read(str(hpf / (k + ".wav")))
        _, y = wavfile.read(str(tmp_path / "wav_nwf" / (k + ".wav")))
        assert np.array_equal(y, MLSA.noise_shaping_one(x, -coef, 0.41))
    # stage 6: restoration, with the high-passed wavs standing in for decoded ones
    out = tmp_path / "decoded"
    out.mkdir()
    for k in names:
        _, x = wavfile.read(str(hpf / (k + ".wav")))
        wavfile.write(str(out / (k + ".wav")), 16000, x)
    dl = out / "wav.scp"
    dl.write_text("".join(str(out / (k + ".wav")) + "\n" for k in names))
    _run(["-m", "pytorchwavenetvocoder_b200.bin.noise_shaping", "--waveforms", str(dl), "--stats", stats, "--outdir",
          str(tmp_path / "decoded_nsf"), "--feature_type", "mcep", "--fs", "16000", "--shiftms", "5", "--mcep_alpha",
          "0.410", "--mag", "0.5", "--n_jobs", "10", "--inv", "false"])
    for k in names:
        _, x = wavfile.read(str(out / (k + ".wav")))
        _, y = wavfile.read(str(tmp_path / "decoded_nsf" / (k + ".wav")))
        assert np.array_equal(y, MLSA.noise_shaping_one(x, coef, 0.41))
