# -*- coding: utf-8 -*-
"""GPU tier of the device-resident corpus: ``wnb_make_train_batch_corpus`` against tests/loader_reference.py applied to
the concatenated stream, bit for bit; ``DeviceCorpusGenerator`` over ``prepare_corpus`` of raw wavs against
``DeviceTrainGenerator`` over the file pipeline's outputs (feature_extract.py melspc and mcep, calc_stats.py twice,
noise_shaping.py), bit for bit, with the same statistics; ``bin/train.py --extract_features true`` against
``bin/train.py`` on the file pipeline's outputs, checkpoint for checkpoint; ``bin/resynthesize.py`` on its result."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import loader_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["f64", "mode0", "mode2", "f32_none"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_make_train_batch_corpus_equals_reference_on_the_stream(mode, seed):
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import encode_mu_law
    from pytorchwavenetvocoder_b200.utils.device_loader import corpus_table
    dt, feat_f64, with_scaler = R.scaler_mode_args(mode)
    rng = np.random.RandomState(seed)
    U, D, N = 80, 20, 9
    frames = rng.randint(0, 40, N) * (rng.rand(N) > 0.2)              # empty utterances and ones shorter than a hop
    frames[0] = max(frames[0], 3)
    lengths = (frames * U).astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    wave16 = rng.randint(-32768, 32768, int(lengths.sum())).astype(np.int16)
    feat = (rng.standard_normal((int(frames.sum()), D)) * 10.0 ** rng.uniform(-2, 2, D)).astype(dt)
    mean = rng.standard_normal(D) * 2 if with_scaler else None
    scale = 0.1 + rng.rand(D) * 3 if with_scaler else None
    orders, order = [], np.arange(N)
    for _ in range(5):
        order = order[rng.permutation(N)]
        orders.append(order)
    L = int(lengths.sum())
    e0 = 1
    starts, offs, begin, end = corpus_table(orders[e0:], e0, lengths, offsets)
    # the stream the table describes, as the ring loader would hold it
    sw = np.concatenate([wave16[offsets[u]:offsets[u] + lengths[u]] for o in orders[e0:] for u in o])
    sf = np.concatenate([feat[offsets[u] // U:(offsets[u] + lengths[u]) // U] for o in orders[e0:] for u in o])
    codes = encode_mu_law((sw / 32768.0).astype(np.float32), 256)
    T, Tf, B = 12 * U, 12, 5
    hop = 7 * U
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    tab = dev(np.stack([starts, offs]))
    d_wave, d_feat, d_mean, d_scale = dev(wave16), dev(feat), dev(mean), dev(scale)
    straddle_utt = straddle_epoch = 0
    for s0 in range(begin, end - (B - 1) * hop - T - 1 + 1, 3 * U):
        x = torch.full((B, T), -1, dtype=torch.int64, device="cuda")
        t = torch.full((B, T), -1, dtype=torch.int64, device="cuda")
        h = torch.full((B, D, Tf), float("nan"), dtype=torch.float32, device="cuda")
        P = _lib.ptr
        _lib.check(_lib.load().wnb_make_train_batch_corpus(
            P(d_wave), P(d_feat), P(tab[0]), P(tab[1]), tab.size(1), begin, end, s0, hop, U, P(d_mean),
            P(d_scale), P(x), P(t), P(h), B, T, Tf, D, feat_f64, 256, _lib.stream()), "make_train_batch_corpus")
        xw, tw, hw = R.make_train_batch(codes, sf, None, s0 - begin, hop, U, len(sw), len(sf), mean, scale, B, T, Tf,
                                        mode)
        assert np.array_equal(x.cpu().numpy(), xw) and np.array_equal(t.cpu().numpy(), tw), s0
        assert np.array_equal(h.cpu().numpy(), hw), s0
        for b in range(B):
            so = s0 + b * hop
            straddle_utt += bool(np.any((starts > so) & (starts <= so + T)))
            straddle_epoch += (so // L) != ((so + T) // L)
    assert straddle_utt > 0 and straddle_epoch > 0


def test_make_train_batch_corpus_rejects_windows_past_the_table():
    from pytorchwavenetvocoder_b200 import _lib
    w = torch.zeros(1600, dtype=torch.int16, device="cuda")
    f = torch.zeros(20, 4, dtype=torch.float32, device="cuda")
    tab = torch.tensor([[0], [0]], dtype=torch.int64, device="cuda")
    x = torch.empty(1, 800, dtype=torch.int64, device="cuda")
    h = torch.empty(1, 4, 10, dtype=torch.float32, device="cuda")
    P = _lib.ptr
    args = lambda s0: (P(w), P(f), P(tab[0]), P(tab[1]), 1, 0, 1600, s0, 80, 80, None, None, P(x), P(x), P(h),  # noqa
                       1, 800, 10, 4, 0, 256, _lib.stream())
    _lib.check(_lib.load().wnb_make_train_batch_corpus(*args(799)), "ok")
    with pytest.raises(_lib.WnbError, match="past the end of the table"):
        _lib.check(_lib.load().wnb_make_train_batch_corpus(*args(800)), "past")
    torch.cuda.synchronize()


# ---- the generator and the statistics against the file pipeline ---------------------------------------------------
def _write_wavs(root, fs, seed):
    from pytorchwavenetvocoder_b200.utils import write_wav_int16
    rng = np.random.RandomState(seed)
    os.makedirs(root)
    names = []
    for i, n in enumerate([9000, 1025, 23456, 4000, 14321, 16000, 7777]):   # ragged, one just over fftl
        k = np.arange(n)
        x = 0.3 * np.sin(k / (3.0 + i)) * np.cos(k / 517.0) + 0.02 * rng.standard_normal(n)
        p = os.path.join(root, "u%d.wav" % i)
        write_wav_int16(p, fs, np.int16(np.clip(x, -1, 1) * 32000))
        names.append(p)
    return sorted(names)


FLAGS = dict(fs=16000, shiftms=5, fftl=1024, mspc_dim=40, highpass_cutoff=70, mcep_dim=24, mcep_alpha=0.41, mag=0.5)


def _file_pipeline(tmp, wavs, ns):
    """the recipe's stages 1-3 through the CLIs: (training wav list, feature list, stats file)"""
    from pytorchwavenetvocoder_b200.bin import calc_stats, feature_extract, noise_shaping
    F = FLAGS
    hdf5, hpf, nwf = os.path.join(tmp, "hdf5"), os.path.join(tmp, "wav_hpf"), os.path.join(tmp, "wav_nwf")
    scp = os.path.join(tmp, "wav.scp")
    open(scp, "w").write("\n".join(wavs) + "\n")
    common = ["--waveforms", scp, "--hdf5dir", hdf5, "--wavdir", hpf, "--fs", str(F["fs"]), "--shiftms",
              str(F["shiftms"]), "--highpass_cutoff", str(F["highpass_cutoff"]), "--fftl", str(F["fftl"])]
    feature_extract.main(common + ["--feature_type", "melspc", "--mspc_dim", str(F["mspc_dim"]), "--fmin", "",
                                   "--fmax", ""])
    if ns:
        feature_extract.main(common + ["--feature_type", "mcep", "--mcep_dim", str(F["mcep_dim"]), "--mcep_alpha",
                                       str(F["mcep_alpha"]), "--save_wav", "false"])
    feats = sorted(os.path.join(hdf5, f) for f in os.listdir(hdf5))
    fscp, stats = os.path.join(tmp, "feats.scp"), os.path.join(tmp, "stats.npz")
    open(fscp, "w").write("\n".join(feats) + "\n")
    calc_stats.main(["--feats", fscp, "--stats", stats, "--feature_type", "melspc"])
    hpf_list = sorted(os.path.join(hpf, f) for f in os.listdir(hpf))
    if not ns:
        return hpf_list, feats, stats
    calc_stats.main(["--feats", fscp, "--stats", stats, "--feature_type", "mcep"])
    hscp = os.path.join(tmp, "wav_hpf.scp")
    open(hscp, "w").write("\n".join(hpf_list) + "\n")
    noise_shaping.main(["--waveforms", hscp, "--stats", stats, "--outdir", nwf, "--feature_type", "mcep", "--fs",
                        str(F["fs"]), "--shiftms", str(F["shiftms"]), "--mcep_alpha", str(F["mcep_alpha"]), "--mag",
                        str(F["mag"]), "--inv", "true"])
    return sorted(os.path.join(nwf, f) for f in os.listdir(nwf)), feats, stats


@pytest.mark.parametrize("ns", [False, True], ids=["plain", "noise_shaping"])
def test_corpus_generator_equals_file_pipeline(tmp_path, ns):
    from pytorchwavenetvocoder_b200.utils import read_hdf5
    from pytorchwavenetvocoder_b200.utils.corpus import prepare_corpus
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceCorpusGenerator, DeviceTrainGenerator
    wavs = _write_wavs(str(tmp_path / "raw"), FLAGS["fs"], 3)
    train_wavs, feats, stats = _file_pipeline(str(tmp_path), wavs, ns)
    F = FLAGS
    corpus = prepare_corpus(wavs, fs=F["fs"], shiftms=F["shiftms"], fftl=F["fftl"], mspc_dim=F["mspc_dim"],
                            highpass_cutoff=F["highpass_cutoff"], noise_shaping=ns, mcep_dim=F["mcep_dim"],
                            mcep_alpha=F["mcep_alpha"], mag=F["mag"], batch_size=3)
    mine = str(tmp_path / "stats_corpus.npz")
    corpus.write_stats(mine)
    with np.load(stats) as a, np.load(mine) as b:
        assert sorted(a.files) == sorted(b.files)
        assert len(a.files) == (6 if ns else 2)
        for k in a.files:
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k
    mean = np.asarray(read_hdf5(stats, "/melspc/mean"))
    scale = np.asarray(read_hdf5(stats, "/melspc/scale"))
    rf, batch_length, B = 1 + 511, 3000, 3
    L = int(corpus.lengths.sum())
    np.random.seed(7)
    devg = DeviceTrainGenerator(train_wavs, feats, rf, batch_length, B, feature_type="melspc", n_quantize=256,
                                mean=mean, scale=scale, shuffle=True, upsampling_factor=corpus.U)
    n_batches = -(-3 * L // (B * devg.hop)) + 2
    devg._utterance(12 * len(wavs))                  # plan past every utterance the readers can reach
    want = [devg.next() for _ in range(n_batches)]
    np.random.seed(7)
    cg = DeviceCorpusGenerator(corpus, rf, batch_length, B, n_quantize=256, mean=corpus.mean, scale=corpus.scale)
    for k, ((xw, hw), tw) in enumerate(want):
        (x, h), t = cg.next()
        assert torch.equal(x, xw) and torch.equal(t, tw), k
        assert torch.equal(h, hw), k
    assert cg.plan.next > 2 * L and cg.stats["tables"] >= 2
    print("%d batches over %.1f epochs, %d table uploads" % (n_batches, cg.plan.next / L, cg.stats["tables"]))


# ---- bin/train.py --extract_features and bin/resynthesize.py -----------------------------------------------------
def _cli(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", module] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=900)
    assert r.returncode == 0, r.stdout.decode()[-3000:]
    return r.stdout.decode()


def test_train_extract_features_equals_file_pipeline(tmp_path):
    wavs = _write_wavs(str(tmp_path / "raw"), FLAGS["fs"], 5)
    train_wavs, feats, stats = _file_pipeline(str(tmp_path), wavs, True)
    F = FLAGS
    model = ["--n_aux", str(F["mspc_dim"]), "--n_resch", "64", "--n_skipch", "128", "--dilation_depth", "4",
             "--dilation_repeat", "2", "--batch_length", "2000", "--batch_size", "2", "--iters", "6", "--intervals", "3",
             "--checkpoint_interval", "3", "--seed", "11", "--feature_type", "melspc"]
    wl, fl = str(tmp_path / "train.scp"), str(tmp_path / "feats.scp")
    open(wl, "w").write("\n".join(train_wavs) + "\n")
    ref, got = str(tmp_path / "exp_files"), str(tmp_path / "exp_corpus")
    _cli("pytorchwavenetvocoder_b200.bin.train", model + ["--waveforms", wl, "--feats", fl, "--stats", stats,
                                                          "--expdir", ref])
    raw = str(tmp_path / "raw")
    _cli("pytorchwavenetvocoder_b200.bin.train", model + [
        "--waveforms", raw, "--expdir", got, "--extract_features", "true", "--fs", str(F["fs"]), "--shiftms",
        str(F["shiftms"]), "--fftl", str(F["fftl"]), "--mspc_dim", str(F["mspc_dim"]), "--fmin", "", "--fmax", "",
        "--highpass_cutoff", str(F["highpass_cutoff"]), "--noise_shaping", "true", "--mcep_dim", str(F["mcep_dim"]),
        "--mcep_alpha", str(F["mcep_alpha"]), "--mag", str(F["mag"])])
    for name in ("checkpoint-3.pkl", "checkpoint-6.pkl", "checkpoint-final.pkl"):
        a = torch.load(os.path.join(ref, name), map_location="cpu", weights_only=False)
        b = torch.load(os.path.join(got, name), map_location="cpu", weights_only=False)
        assert a.keys() == b.keys()
        for k in a["model"]:
            assert torch.equal(a["model"][k], b["model"][k]), (name, k)
        if "optimizer" in a:
            for pid, st in a["optimizer"]["state"].items():
                for kk, v in st.items():
                    assert torch.equal(torch.as_tensor(v), torch.as_tensor(b["optimizer"]["state"][pid][kk])), (name, kk)
    mine = os.path.join(got, "stats.npz" if not _have_h5py() else "stats.h5")
    conf = torch.load(os.path.join(got, "model.conf"), weights_only=False)
    assert conf.extract_features and conf.noise_shaping and conf.mspc_dim == F["mspc_dim"]
    from pytorchwavenetvocoder_b200.utils import read_hdf5
    for key in ("/melspc/mean", "/melspc/scale", "/mcep/mean", "/mcep/scale", "/mlsa/coef", "/mlsa/alpha"):
        assert np.array_equal(read_hdf5(mine, key), read_hdf5(stats, key)), key
    # the decoding side takes the written statistics unchanged
    out = str(tmp_path / "resyn")
    _cli("pytorchwavenetvocoder_b200.bin.resynthesize", [
        "--waveforms", str(tmp_path / "raw"), "--checkpoint", os.path.join(got, "checkpoint-final.pkl"), "--outdir",
        out, "--stats", mine, "--noise_shaping", "--fs", str(F["fs"]), "--fmin", "", "--fmax", "", "--batch_size", "7"])
    assert sorted(os.listdir(out)) == sorted(os.path.basename(w) for w in wavs)


def _have_h5py():
    try:
        import h5py  # noqa: F401
        return True
    except ImportError:
        return False
