# -*- coding: utf-8 -*-
"""GPU tier: continuous batching on the fp32 streaming decoder (``WaveNet.decode_pool(..., kernel="stream")``) is
bit-identical to one-shot streaming decoding.

Stream k of a ``kernel="stream"`` pool with seed S must equal row k of ``net._decode(X, H, n_list, mode, seed=S,
kernel="stream")`` (``torch.equal``) for any one-shot batch size: the streaming decoder's sums do not depend on its launch
form.  Covered: 64/64 at ks 2 and ks 3 with aux at frame rate (U 4), a speaker-code shape (U 0, A 31) and arctic
512/256 at few samples; argmax and Philox sampling; seeds of 1 sample and longer than the receptive field; streams
admitted in different calls, in lock step and with ``park_below`` 1 and m; capacities that put the decoder at NU 1, 2
and 4; cancels; ``step_pcm16``; the library launches of a steady, an admitting and a parking + resuming call; the
refusals; and ``bin/decode.py --pool_capacity`` under fp32 at a shape outside the warp decoder."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS2_U = (256, 28, 64, 64, 4, 2, 2, 4)
KS3_U = (256, 28, 64, 64, 4, 2, 3, 4)
SPEAKER = (256, 31, 64, 64, 4, 2, 2, 0)
ARCTIC = (256, 28, 512, 256, 10, 3, 2, 80)
_MODELS = {}


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 91 + len(_MODELS))).eval()
        assert net.decode_math == "fp32"
        _MODELS[t] = net
    return _MODELS[t]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _streams(net, n, seed, lengths=(30, 301), arrivals=20):
    """n streams: seed codes, length, aux frames (A, nf) on the GPU, arrival call"""
    rng = np.random.RandomState(seed)
    rf, U = net.receptive_field, max(net.upsampling_factor, 1)
    out = []
    for k in range(n):
        T0 = [1, 2 * rf + 7][k % 2]
        total = int(rng.randint(*lengths))
        nf = (T0 - 1 + total + U - 1) // U + 1
        x = torch.from_numpy(rng.randint(0, net.n_quantize, size=T0)).cuda()
        h = torch.from_numpy(rng.standard_normal((net.n_aux, nf)).astype(np.float32)).cuda()
        out.append((x, total, h, int(rng.randint(0, arrivals))))
    return out


def _one_shot(net, streams, mode, seed, B=None):
    """{k: codes of stream k} from one-shot streaming decodes of B rows (default: one row per stream), one per seed
    length, stream k in row k"""
    N, A, U = len(streams), net.n_aux, max(net.upsampling_factor, 1)
    B = B or N
    nfmax = (max(x.numel() for x, _, _, _ in streams) - 1 + max(n for _, n, _, _ in streams) + U - 1) // U + 1
    H = torch.zeros(B, A, nfmax, device="cuda")
    for k, (_, _, h, _) in enumerate(streams):
        H[k, :, :h.size(1)] = h
    n_list = [total for _, total, _, _ in streams] + [1] * (B - N)
    want = {}
    for T0 in sorted({x.numel() for x, _, _, _ in streams}):
        X = torch.zeros(B, T0, dtype=torch.int64, device="cuda")
        for k, (x, _, _, _) in enumerate(streams):
            if x.numel() == T0:
                X[k] = x
        with torch.no_grad():
            gen = net._decode(X, H, n_list, mode, seed=seed, kernel="stream").cpu()
        assert net.last_decode_kernel == "stream"
        for k, (x, total, _, _) in enumerate(streams):
            if x.numel() == T0:
                want[k] = gen[k, :total]
    return want


def _run_pool(net, streams, capacity, mode, seed, rng_seed, park_below=None, cancel_after=None, stall=0.0):
    """Drive a stream pool: streams arrive at their call and are fed random chunks; with ``stall`` a stream gets no
    frames in that share of the calls.  Stream k is cancelled once it has cancel_after[k] samples."""
    rng = np.random.RandomState(rng_seed)
    cancel_after = cancel_after or {}
    Uc = max(net.upsampling_factor, 1)
    pool = net.decode_pool(capacity, mode, seed, park_below=park_below, kernel="stream")
    assert pool.kernel == "stream"
    got = {k: [] for k in range(len(streams))}
    sent = [0] * len(streams)
    it = 0
    while it <= max(a for _, _, _, a in streams) or not all(pool.finished(k) for k in range(len(streams))):
        for k, (x, total, h, arrival) in enumerate(streams):
            if arrival == it:
                F = int(rng.randint(0, 3))
                assert pool.admit(x, total, h[:, :F] if F else None, stream=k) == k
                sent[k] = F
            elif arrival < it and not pool.finished(k) and sent[k] < h.size(1) and rng.rand() >= stall:
                F = min(int(rng.randint(0, 120 // Uc + 2)), h.size(1) - sent[k])
                pool.feed(k, h[:, sent[k]:sent[k] + F])
                sent[k] += F
        it += 1
        for k, codes in pool.step(None if rng.rand() < 0.2 else int(rng.randint(1, 150))).items():
            got[k].append(codes.cpu())
        for k, n in cancel_after.items():
            if k in pool.active + pool.parked and sum(c.numel() for c in got[k]) >= n:
                pool.cancel(k)
    return pool, {k: torch.cat(v) if v else torch.empty(0, dtype=torch.int32) for k, v in got.items()}


def _check(got, want, what):
    for k in want:
        assert torch.equal(got[k], want[k]), (what, k, int((got[k] != want[k]).sum()))


SHAPES = {"ks2_u4": KS2_U, "ks3_u4": KS3_U, "speaker_A31_U0": SPEAKER}


@pytest.mark.parametrize("park_below", [None, 1, 40])
@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_pool_equals_one_shot(shape, mode, park_below):
    net = _model(SHAPES[shape])
    si = list(SHAPES).index(shape)
    streams = _streams(net, 24, 30 + si)
    seed = 3000 + si
    want = _one_shot(net, streams, mode, seed)
    pool, got = _run_pool(net, streams, 8, mode, seed, 11 + si, park_below, stall=0.0 if park_below is None else 0.3)
    assert not pool.active and not pool.waiting and not pool.parked
    _check(got, want, (shape, mode, park_below))


def test_arctic_pool_equals_one_shot():
    net = _model(ARCTIC)
    streams = _streams(net, 6, 8, lengths=(10, 60), arrivals=3)
    want = _one_shot(net, streams, "sampling", 41)
    _, got = _run_pool(net, streams, 4, "sampling", 41, 2)
    _check(got, want, "arctic")


@pytest.mark.parametrize("which", ["nu1", "nu2", "nu4"])
def test_capacities(which):
    """a pool of sms - 1, sms + 1 and 2 sms + 1 rows (the decoder's NU 1, 2 and 4) against one-shot batches of another
    size"""
    net = _model(KS2_U)
    sms = _sms()
    capacity = {"nu1": sms - 1, "nu2": sms + 1, "nu4": 2 * sms + 1}[which]
    streams = _streams(net, 40, 50 + capacity, lengths=(20, 121), arrivals=6)
    want = _one_shot(net, streams, "sampling", 77, B=len(streams) + 3)
    _, got = _run_pool(net, streams, capacity, "sampling", 77, 5)
    _check(got, want, which)


def test_cancel():
    net = _model(KS3_U)
    streams = _streams(net, 16, 17)
    want = _one_shot(net, streams, "sampling", 9)
    cancel_after = {3: 0, 7: 60, 12: 10}
    pool, got = _run_pool(net, streams, 6, "sampling", 9, 21, 8, cancel_after, stall=0.3)
    for k in range(len(streams)):
        assert pool.finished(k)
        if k in cancel_after:
            assert torch.equal(got[k], want[k][:got[k].numel()]), k
        else:
            assert torch.equal(got[k], want[k]), k


def test_launch_counts():
    """steady call: the inputs kernel and the decode (2); admitting call (one group, L layers): the prefill's front and
    L - 1 layer launches, one move, the inputs kernel and the decode (L + 3); a call that parks one stream and resumes
    another: one move each way and the two (4); a call with nothing to run: none"""
    from pytorchwavenetvocoder_b200 import _lib
    net = _model(KS3_U)
    L = len(net.dilations)
    pool = net.decode_pool(8, "sampling", 3, park_below=1, kernel="stream")
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    h = torch.randn(28, 400, device="cuda")
    pool.admit(x, 1000, h[:, :40])
    pool.admit(x, 1000, h[:, :40])

    def call():
        l0 = _lib.launch_count()
        out = pool.step()
        torch.cuda.synchronize()
        return _lib.launch_count() - l0, sorted(out)

    assert call() == (L + 3, [0, 1])
    assert call() == (0, [])
    pool.feed(1, h[:, 40:80])
    assert call() == (3, [1]) and pool.parked == [0]
    pool.feed(0, h[:, 40:80])
    assert call() == (4, [0]) and pool.parked == [1]
    pool.feed(0, h[:, 80:120])
    pool.feed(1, h[:, 80:120])
    pool.step()                               # resumes 1
    pool.feed(0, h[:, 120:160])
    pool.feed(1, h[:, 120:160])
    assert call() == (2, [0, 1])


def test_step_pcm16_equals_codes():
    from pytorchwavenetvocoder_b200.nets.wavenet import codes_to_pcm16
    net = _model(KS2_U)
    streams = _streams(net, 3, 5)
    want = _one_shot(net, streams, "sampling", 4)
    pool = net.decode_pool(4, "sampling", 4, kernel="stream")
    got = {k: [] for k in range(3)}
    for k, (x, total, h, _) in enumerate(streams):
        pool.admit(x, total, h)
    while pool.active or pool.waiting:
        for k, pcm in pool.step_pcm16(64).items():
            got[k].append(pcm.cpu())
    for k in range(3):
        assert torch.equal(torch.cat(got[k]), codes_to_pcm16(want[k].cuda(), 256).cpu()), k


def test_errors():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import WaveNet
    net = _model(KS3_U)
    with pytest.raises(_lib.WnbError, match="warp decoder"):
        net.decode_pool(8)                                              # "auto" under fp32 stays on the warp decoder
    with pytest.raises(_lib.WnbError, match="warp decoder"):
        net.decode_pool(8, kernel="warp")
    with pytest.raises(_lib.WnbError, match="streaming decoder"):
        WaveNet(256, 28, 64, 62, 2, 1, 2, 0).cuda().decode_pool(8, kernel="stream")    # S 62: not a multiple of 4
    with pytest.raises(_lib.WnbError, match="streaming decoder"):
        WaveNet(256, 28, 1024, 64, 1, 1, 2, 0).cuda().decode_pool(8, kernel="stream")  # R 1024: 512 lanes
    with pytest.raises(_lib.WnbError):
        net.decode_pool(8, kernel="bf16")                               # bf16 kernel under fp32 math
    with pytest.raises(ValueError):
        net.decode_pool(8, kernel="direct")
    assert net.decode_pool(8, kernel="stream").kernel == "stream"


# ---- bin/decode.py --pool_capacity ---------------------------------------------------------------------------------
def _cli(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.decode"] + args, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    assert r.returncode == 0, r.stdout.decode()[-3000:]


@pytest.mark.parametrize("gpus", [1, 2])
def test_cli_pool_writes_the_pool_api_files(tmp_path, gpus):
    """decode.py --pool_capacity 8 under fp32 at 64/64 ks 3 (outside the warp decoder) writes the wavs of a direct
    kernel="stream" pool run with the worker's drawn seed, with and without --noise_shaping"""
    from pytorchwavenetvocoder_b200.bin import decode as D
    from pytorchwavenetvocoder_b200.nets import WaveNet, codes_to_pcm16, decode_mu_law
    from pytorchwavenetvocoder_b200.utils import have_soundfile, write_hdf5, write_wav, write_wav_pcm16
    from pytorchwavenetvocoder_b200.utils.mlsa import convert_mcep_to_mlsa_coef, mlsa_filter_batch
    if gpus > torch.cuda.device_count():
        pytest.skip("needs %d GPUs" % gpus)
    U, D_, R, S, depth, ks = 16, 28, 64, 64, 4, 3
    rng = np.random.RandomState(12)
    torch.manual_seed(0)
    net = WaveNet(256, D_, R, S, depth, 2, ks, U)
    expdir, featdir = tmp_path / "exp", tmp_path / "feats"
    expdir.mkdir()
    featdir.mkdir()
    ckpt = str(expdir / "checkpoint-final.pkl")
    torch.save({"model": net.state_dict()}, ckpt)
    conf = argparse.Namespace(n_quantize=256, n_aux=D_, n_resch=R, n_skipch=S, dilation_depth=depth, dilation_repeat=2,
                              kernel_size=ks, upsampling_factor=U, use_upsampling_layer=True, feature_type="world",
                              use_speaker_code=False)
    torch.save(conf, str(expdir / "model.conf"))
    nfs = [20, 41, 33, 27, 50, 38, 22, 45, 31, 36, 29]
    feats, hs = [], []
    for i, nf in enumerate(nfs):
        f = str(featdir / ("p%02d.npz" % i))
        h = rng.standard_normal((nf, D_))
        write_hdf5(f, "/world", h)
        feats.append(f)
        hs.append(h)
    fl, stats = str(tmp_path / "feats.scp"), str(tmp_path / "stats.npz")
    open(fl, "w").write("\n".join(feats) + "\n")
    write_hdf5(stats, "/world/mean", np.zeros(D_))
    write_hdf5(stats, "/world/scale", np.ones(D_))
    coef = convert_mcep_to_mlsa_coef(rng.randn(25) * 0.5, 0.5, 0.41)
    write_hdf5(stats, "/mlsa/coef", coef)
    write_hdf5(stats, "/mlsa/alpha", 0.41)
    common = ["--feats", fl, "--checkpoint", ckpt, "--stats", stats, "--fs", "16000", "--seed", "5", "--n_gpus",
              str(gpus), "--decode_math", "fp32", "--pool_capacity", "8", "--batch_size", "3"]
    plain, shaped = str(tmp_path / "plain"), str(tmp_path / "shaped")
    _cli(common + ["--outdir", plain])
    _cli(common + ["--outdir", shaped, "--noise_shaping"])
    net = net.cuda().eval()
    assert D.pool_kernel_for(net, 8) == "stream"
    scaler = D.load_scaler(stats, "world")
    for gpu, idx in enumerate(np.array_split(np.arange(len(feats)), gpus)):
        seed = D.pool_seed(5, gpu)
        with torch.no_grad():
            pool = net.decode_pool(8, "sampling", seed, kernel="stream")
            for j, i in enumerate(idx):
                ht = torch.from_numpy(scaler.transform(hs[i])).float().t().contiguous().cuda()
                pool.admit(torch.full((1,), 128, dtype=torch.int64, device="cuda"), nfs[i] * U - 1, ht, stream=j)
            got = {j: [] for j in range(len(idx))}
            while pool.active or pool.waiting:
                for j, c in pool.step().items():
                    got[j].append(c)
        for j, i in enumerate(idx):
            codes = torch.cat(got[j])
            assert codes.numel() == nfs[i] * U - 1
            name = "p%02d.wav" % i
            want = str(tmp_path / ("want_" + name))
            if have_soundfile():
                write_wav(want, decode_mu_law(codes.cpu().numpy().astype(np.int64), 256), 16000)
            else:
                write_wav_pcm16(want, codes_to_pcm16(codes, 256).cpu().numpy(), 16000)
            assert open(os.path.join(plain, name), "rb").read() == open(want, "rb").read(), (gpus, i)
            pcm = codes_to_pcm16(codes, 256).cpu().numpy()
            write_wav_pcm16(want, mlsa_filter_batch([pcm], coef, 0.41, 4)[0], 16000)
            assert open(os.path.join(shaped, name), "rb").read() == open(want, "rb").read(), (gpus, i)
