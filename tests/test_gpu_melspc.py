# -*- coding: utf-8 -*-
"""GPU tier: the melspc features (csrc/melspc.cu, DESIGN.md §6 row f5) against the float64 restatement of
tests/melspc_reference.py, element by element.

Bars (derivations in ``melspc_reference.feature_bounds`` and ``fir_bound``):
  * float32 features: each equals ``np.float32(oracle64)``, except where the interval of ``feature_bounds`` around the
    oracle's float64 value straddles a float32 rounding boundary, and there it is one of the two neighbours;
  * the filtered float64 signal: within sum_k |b_k x_{n-k}| * 255 * 2^-53 of the oracle's;
  * the filtered int16 wav: ``np.int16(oracle)``, except where the oracle lies within that bound of an integer.
Then ragged batches, int16 / float64 input, cutoff 70 / 0, fftl 64 ... 4096, hops 80 / 110 / 256, 80 / 40 mels, fmin /
fmax, digital silence, full-scale square waves, the full-size batch (64 x 160 000), unsupported fftl, determinism, and
the recipe's stages 1, 2, 4 and 5 end to end through the CLIs."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import melspc_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAGGED = [1, 2, 511, 512, 513, 1023, 1024, 1025, 16000, 160000]


def _speechlike(rng, n, amp=8000.0):
    x = np.cumsum(rng.randn(n))
    x -= np.linspace(x[0], x[-1], n)
    x = x / (np.abs(x).max() + 1e-9) * amp + rng.randn(n) * 30.0 + 200.0 * np.sin(np.arange(n) * 0.013)
    return x


def _check_features(xs, fs, fftl, hop, n_mels, fmin=None, fmax=None, cutoff=0, which=None, label=""):
    """Run melspc_batch on the whole list and compare the utterances in ``which`` (default all) with the oracle; also
    the filtered float64 signal and int16 wav when there is a cutoff.  Returns (exact, total) feature counts."""
    from pytorchwavenetvocoder_b200.utils.melspc import lowcut_filter_batch, lowcut_taps, melspc_batch
    out = melspc_batch(xs, fs, fftl, hop, n_mels, fmin, fmax, cutoff, filtered_int16=bool(cutoff))
    feats, wavs = out if cutoff else (out, None)
    yf = lowcut_filter_batch(xs, fs, cutoff)[0] if cutoff else None
    taps = lowcut_taps(fs, cutoff) if cutoff else None
    exact = total = 0
    for u in (range(len(xs)) if which is None else which):
        want, E, xf, mag = R.melspc(xs[u], fs, fftl, hop, n_mels, fmin, fmax, taps)
        got = feats[u]
        where = "%s utterance %d (length %d)" % (label, u, len(xs[u]))
        assert got.dtype == np.float32 and got.shape == want.shape, (where, got.shape, want.shape)
        delta = R.fir_bound(mag)
        if cutoff:
            err = np.abs(yf[u] - xf)
            if not np.all(err <= delta):
                n = int(np.argmax(err > delta))
                raise AssertionError("%s: filtered sample %d: GPU %r, oracle %r, |diff| %.3g > bound %.3g"
                                     % (where, n, yf[u][n], xf[n], err[n], delta[n]))
            from pytorchwavenetvocoder_b200.utils.melspc import int16_cast
            near = np.abs(xf - np.round(xf)) <= delta
            ok16 = (wavs[u] == np.int16(int16_cast(xf))) | (near & ((wavs[u] == int16_cast(xf - delta)) |
                                                                    (wavs[u] == int16_cast(xf + delta))))
            if not ok16.all():
                n = int(np.argmin(ok16))
                raise AssertionError("%s: int16 wav sample %d: GPU %d, oracle np.int16(%r) = %d"
                                     % (where, n, wavs[u][n], xf[n], int16_cast(xf[n:n + 1])[0]))
        lo, hi = R.feature_bounds(xf, delta, E, fs, fftl, hop, n_mels, fmin, fmax)
        ok = (got >= np.float32(lo)) & (got <= np.float32(hi))
        if not ok.all():
            t, m = np.argwhere(~ok)[0]
            raise AssertionError("%s: frame %d, mel %d: GPU %r, np.float32(oracle) %r (oracle64 %r, E %r), allowed "
                                 "[%r, %r]; %d elements outside" % (where, t, m, got[t, m], want[t, m],
                                                                    np.log10(max(E[t, m], R.EPS)), E[t, m],
                                                                    np.float32(lo[t, m]), np.float32(hi[t, m]),
                                                                    int((~ok).sum())))
        exact += int((got == want).sum())
        total += got.size
    print("%s: %d / %d features equal np.float32(oracle64) (%.6f %%)" % (label, exact, total, 100.0 * exact / total))
    return exact, total


def test_ragged_int16_lowcut_arctic():
    rng = np.random.RandomState(0)
    xs = [np.int16(_speechlike(rng, n)) if n > 2 else np.int16(rng.randn(n) * 3000) for n in RAGGED]
    exact, total = _check_features(xs, 16000, 1024, 80, 80, cutoff=70, label="arctic int16 cutoff 70")
    assert exact >= 0.999 * total


def test_ragged_float64_no_cutoff_fftl256_hop110_40mels():
    rng = np.random.RandomState(1)
    xs = [_speechlike(rng, n, 12000.0) if n > 2 else rng.randn(n) * 3000 for n in RAGGED]
    _check_features(xs, 16000, 256, 110, 40, label="float64 fftl 256 hop 110")


@pytest.mark.parametrize("fftl,hop,n_mels,fs,fmin,fmax,cutoff", [
    (64, 80, 40, 16000, None, None, 70),
    (4096, 256, 80, 22050, 125, 7600, 70),
    (1024, 256, 80, 22050, None, None, 70),      # ljspeech
    (1024, 80, 80, 16000, 80, 7600, 0),
    (2048, 110, 40, 24000, None, 9000, 0),
])
def test_fftl_hop_mels_and_band_limits(fftl, hop, n_mels, fs, fmin, fmax, cutoff):
    rng = np.random.RandomState(fftl + hop)
    lens = [1, 2, fftl // 2 - 1, fftl // 2, fftl // 2 + 1, fftl - 1, fftl, fftl + 1, 3 * fftl + 7, 16000]
    xs = [np.int16(_speechlike(rng, n)) if n > 2 else np.int16(rng.randn(n) * 3000) for n in lens]
    _check_features(xs, fs, fftl, hop, n_mels, fmin, fmax, cutoff, label="fftl %d hop %d" % (fftl, hop))


def test_digital_silence_is_log10_eps():
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    floor = np.float32(np.log10(1e-10))
    for cutoff in (70, 0):
        xs = [np.zeros(n, dtype=np.int16) for n in (1, 700, 16000)]
        out = melspc_batch(xs, 16000, 1024, 80, 80, highpass_cutoff=cutoff, filtered_int16=bool(cutoff))
        feats = out[0] if cutoff else out
        for f in feats:
            assert np.all(f == floor), (cutoff, f[f != floor][:5])
        if cutoff:
            assert all(not w.any() for w in out[1])


def test_full_scale_square_waves_wrap_int16():
    """A full-scale square wave through the low-cut filter overshoots int16 (sum |b| = 1.87); the wav keeps np.int16's
    wrap-around, and the features still follow the oracle."""
    from pytorchwavenetvocoder_b200.utils.melspc import lowcut_filter_batch
    xs = [np.int16(np.where((np.arange(n) // p) % 2 == 0, 32767, -32768)) for n, p in ((8000, 50), (12345, 173),
                                                                                     (3000, 9))]
    _check_features(xs, 16000, 1024, 80, 80, cutoff=70, label="square waves")
    y, y16 = lowcut_filter_batch(xs, 16000, 70)
    assert max(np.abs(v).max() for v in y) > 32768           # the filtered signal does overshoot
    assert any(np.any((np.abs(v) > 32768) & (np.sign(w) != np.sign(v)) & (w != 0)) for v, w in zip(y, y16))


def test_full_size_batch_three_utterances_exact():
    """64 utterances of 160 000 samples (10 s at 16 kHz) in one launch per stage; three compared element by element."""
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    rng = np.random.RandomState(4)
    xs = [np.int16(_speechlike(rng, 160000 - (i % 5) * 37)) for i in range(64)]
    _check_features(xs, 16000, 1024, 80, 80, cutoff=70, which=(0, 31, 63), label="64 x 160 000")
    feats = melspc_batch(xs, 16000, 1024, 80, 80, highpass_cutoff=70)
    assert all(f.shape == (1 + len(x) // 80, 80) and np.isfinite(f).all() for f, x in zip(feats, xs))


def test_unsupported_fftl_raises():
    from pytorchwavenetvocoder_b200._lib import WnbError
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    xs = [np.int16(np.arange(5000) % 300)]
    for fftl in (1000, 8192, 32):
        with pytest.raises(WnbError, match="fftl %d is not supported" % fftl):
            melspc_batch(xs, 16000, fftl, 80, 80, highpass_cutoff=70)


def test_two_runs_bit_identical():
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    rng = np.random.RandomState(5)
    xs = [np.int16(_speechlike(rng, n)) for n in (16000, 513, 48000)]
    a = melspc_batch(xs, 16000, 1024, 80, 80, highpass_cutoff=70, filtered_int16=True)
    b = melspc_batch(xs, 16000, 1024, 80, 80, highpass_cutoff=70, filtered_int16=True)
    for fa, fb in zip(a[0] + a[1], b[0] + b[1]):
        assert np.array_equal(fa.view(np.uint8), fb.view(np.uint8))


def _run(args, timeout=600):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout)
    assert r.returncode == 0, r.stdout.decode()[-3000:]
    return r.stdout.decode()


def test_recipe_stages_end_to_end(tmp_path):
    """egs/arctic/sd-melspc stages 1, 2, 4 and 5 with its flags: wavs -> bin/feature_extract.py (features + filtered
    wavs, equal to melspc_batch) -> bin/calc_stats.py -> bin/train.py --feature_type melspc (two iterations of a small
    model) -> bin/decode.py of one utterance."""
    from scipy.io import wavfile
    from pytorchwavenetvocoder_b200.utils import read_hdf5, read_wav
    from pytorchwavenetvocoder_b200.utils.melspc import melspc_batch
    rng = np.random.RandomState(6)
    wavdir, hpf, h5 = tmp_path / "wav", tmp_path / "wav_hpf", tmp_path / "hdf5"
    wavdir.mkdir()
    xs = {}
    for i, n in enumerate((16000, 12345, 20000)):
        xs["u%d" % i] = np.int16(_speechlike(rng, n, 9000.0))
        wavfile.write(str(wavdir / ("u%d.wav" % i)), 16000, xs["u%d" % i])
    scp = tmp_path / "wav.scp"
    scp.write_text("".join(str(wavdir / ("u%d.wav" % i)) + "\n" for i in range(3)))
    _run(["-m", "pytorchwavenetvocoder_b200.bin.feature_extract", "--waveforms", str(scp), "--wavdir", str(hpf),
          "--hdf5dir", str(h5), "--feature_type", "melspc", "--fs", "16000", "--shiftms", "5", "--mspc_dim", "80",
          "--highpass_cutoff", "70", "--fftl", "1024", "--fmin", "", "--fmax", "", "--n_jobs", "10", "--batch_size",
          "2"])
    names = sorted(xs)
    feats, wavs = melspc_batch([xs[k] for k in names], 16000, 1024, 80, 80, highpass_cutoff=70, filtered_int16=True)
    files = []
    for k, f, w in zip(names, feats, wavs):
        ff = (glob.glob(str(h5 / (k + ".h5"))) + glob.glob(str(h5 / (k + ".npz"))))[0]
        files.append(ff)
        assert np.array_equal(read_hdf5(ff, "/melspc"), f)
        fs, y = wavfile.read(str(hpf / (k + ".wav")))
        assert fs == 16000 and y.dtype == np.int16 and np.array_equal(y, w)
    fl, wl = tmp_path / "feats.scp", tmp_path / "wav_hpf.scp"
    fl.write_text("".join(f + "\n" for f in files))
    wl.write_text("".join(str(hpf / (k + ".wav")) + "\n" for k in names))
    stats = str(tmp_path / "stats.npz")
    _run(["-m", "pytorchwavenetvocoder_b200.bin.calc_stats", "--feats", str(fl), "--stats", stats, "--feature_type",
          "melspc"])
    assert read_hdf5(stats, "/melspc/mean").shape == (80,)
    expdir = str(tmp_path / "exp")
    log = _run(["-m", "pytorchwavenetvocoder_b200.bin.train", "--waveforms", str(wl), "--feats", str(fl), "--stats",
                stats, "--expdir", expdir, "--feature_type", "melspc", "--n_aux", "80", "--n_resch", "64",
                "--n_skipch", "64", "--dilation_depth", "4", "--dilation_repeat", "1", "--upsampling_factor", "80",
                "--batch_length", "800", "--batch_size", "2", "--iters", "2", "--intervals", "1",
                "--checkpoint_interval", "2", "--verbose", "1"])
    assert "average loss" in log and os.path.exists(expdir + "/checkpoint-final.pkl")
    one = tmp_path / "one.scp"
    one.write_text(files[1] + "\n")
    outdir = str(tmp_path / "out")
    _run(["-m", "pytorchwavenetvocoder_b200.bin.decode", "--feats", str(one), "--checkpoint",
          expdir + "/checkpoint-final.pkl", "--stats", stats, "--outdir", outdir, "--fs", "16000", "--batch_size", "1",
          "--intervals", "1000"])
    x, fs = read_wav(os.path.join(outdir, "u1.wav"))
    assert fs == 16000 and len(x) == feats[1].shape[0] * 80 - 1
