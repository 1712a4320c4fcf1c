# -*- coding: utf-8 -*-
"""GPU tier: continuous batching on the fp32 warp decoder (``WaveNet.decode_pool`` with ``decode_math="fp32"``) is
bit-identical to one-shot warp decoding at the pool's launch form.

Stream k of an fp32 pool with seed S must equal row k of ``net._decode(X, H, n_list, mode, seed=S, kernel="warp")``
(``torch.equal``) for a one-shot batch whose warp form (``wnb_decode_warp_form``: NU, W, CL) equals the pool's; the
one-shot batch is padded with one-sample rows up to a size of that form.  Covered: the 64/512 shape with 30 layers (U 80),
a 10-layer 64/512 and a speaker-code shape (U 0, A 31), in argmax and Philox sampling, with seeds of 1 sample, rf + 2 000
and 5 rf + 3 in one pool, aux frames in random chunks, random ``max_samples`` windows and rows reused; every form the
card reaches (CL 2 at 8 and 64 rows, CL 1 at sms/2 + 1 rows, NU 2 at sms + 1 rows); the queues an admission leaves in
a CL 1 pool, bit for bit against a CL 1 prefill and unlike a CL 2 one (the prefill must run at the pool's CL, not at
the CL a group smaller than sms/2 would get on its own, and codes alone would rarely show the difference); parking under ``park_below``
1 and 80 with stalls, cancels and a counter rebase; ``wnb_decode_pool_move`` against ``torch.roll``; the library launches
of a steady, an admitting and a parking + resuming call; ``step_pcm16``; and ``bin/decode.py --pool_capacity``."""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.test_gpu_decode_pool_park import _moves, _run_parking_pool, _trace
from tests.util import our_model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE30 = (256, 28, 64, 512, 10, 3, 2, 80)
SHALLOW10 = (256, 28, 64, 512, 10, 1, 2, 80)
SPEAKER = (256, 31, 64, 512, 4, 2, 2, 0)
_MODELS = {}


def _model(t):
    if t not in _MODELS:
        cfg = O.Config(*t)
        net = our_model(cfg, O.make_params(cfg, 71 + len(_MODELS))).eval()
        assert net.decode_math == "fp32"
        _MODELS[t] = (cfg, net)
    return _MODELS[t]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _form(B, L):
    from pytorchwavenetvocoder_b200 import _lib
    f = (ctypes.c_int32 * 4)()
    _lib.check(_lib.load().wnb_decode_warp_form(B, L, f), "decode_warp_form")
    return tuple(f[:3])


def _streams(cfg, n, seed, lengths=(50, 401), arrivals=40):
    """n streams: seed codes, length, aux frames (A, nf) on the GPU, arrival call"""
    rng = np.random.RandomState(seed)
    rf, U = cfg.receptive_field, max(cfg.upsampling_factor, 1)
    out = []
    for k in range(n):
        T0 = [1, rf + 2000, 5 * rf + 3][k % 3]
        total = int(rng.randint(*lengths))
        nf = (T0 - 1 + total + U - 1) // U + 1
        x = torch.from_numpy(rng.randint(0, cfg.n_quantize, size=T0)).cuda()
        h = torch.from_numpy(rng.standard_normal((cfg.n_aux, nf)).astype(np.float32)).cuda()
        out.append((x, total, h, int(rng.randint(0, arrivals))))
    return out


def _one_shot(net, streams, mode, seed, capacity):
    """{k: codes of stream k} from one-shot warp decodes at the pool's form, one per seed length, stream k in row k"""
    N, A, U, L = len(streams), net.n_aux, max(net.upsampling_factor, 1), len(net.dilations)
    form = _form(capacity, L)
    B = next(b for b in range(N, 8 * capacity + 1) if _form(b, L) == form)
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
            gen = net._decode(X, H, n_list, mode, seed=seed, kernel="warp").cpu()
        for k, (x, total, _, _) in enumerate(streams):
            if x.numel() == T0:
                want[k] = gen[k, :total]
    return want


def _run_pool(net, streams, capacity, mode, seed, rng_seed):
    rng = np.random.RandomState(rng_seed)
    pool = net.decode_pool(capacity, mode, seed)
    got = {k: [] for k in range(len(streams))}
    sent = [0] * len(streams)
    it = 0
    while it <= max(a for _, _, _, a in streams) or not all(pool.finished(k) for k in range(len(streams))):
        for k, (x, total, h, arrival) in enumerate(streams):
            if arrival == it:
                F = int(rng.randint(0, 3))
                assert pool.admit(x, total, h[:, :F] if F else None, stream=k) == k
                sent[k] = F
            elif arrival < it and not pool.finished(k) and sent[k] < h.size(1):
                F = min(int(rng.randint(0, 40)), h.size(1) - sent[k])
                pool.feed(k, h[:, sent[k]:sent[k] + F])
                sent[k] += F
        it += 1
        for k, codes in pool.step(None if rng.rand() < 0.2 else int(rng.randint(1, 150))).items():
            got[k].append(codes.cpu())
    return pool, {k: torch.cat(v) for k, v in got.items()}


def _check(got, want, what):
    for k in want:
        assert torch.equal(got[k], want[k]), (what, k, int((got[k] != want[k]).sum()))


SHAPES = {"base_L30": BASE30, "shallow_L10": SHALLOW10, "speaker_A31_U0": SPEAKER}


@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_pool_equals_one_shot(shape, mode):
    cfg, net = _model(SHAPES[shape])
    si = list(SHAPES).index(shape)
    streams = _streams(cfg, 40, 30 + si)
    seed = 3000 + si
    want = _one_shot(net, streams, mode, seed, 8)
    pool, got = _run_pool(net, streams, 8, mode, seed, 11 + si)
    assert not pool.active and not pool.waiting
    _check(got, want, (shape, mode))


@pytest.mark.parametrize("which", ["cl2_64", "cl1", "nu2"])
def test_every_form(which, monkeypatch):
    """64 rows (CL 2), sms/2 + 1 (CL 1, one utterance per CTA) and sms + 1 (two per CTA), with short streams.  Every
    admission group of the CL 1 pool is smaller than sms/2, where the group alone would run the 2-CTA form."""
    cfg, net = _model(BASE30)
    L, sms = len(cfg.dilations), _sms()
    capacity, n = {"cl2_64": (64, 60), "cl1": (sms // 2 + 1, sms), "nu2": (sms + 1, sms + sms // 2)}[which]
    form = _form(capacity, L)
    assert form == {"cl2_64": (1, 16, 2), "cl1": (1, 16, 1), "nu2": (2, 16, 1)}[which], form
    streams = _streams(cfg, n, 50 + capacity, lengths=(20, 121), arrivals=12)
    want = _one_shot(net, streams, "sampling", 77, capacity)
    calls = _trace(monkeypatch)
    pool, got = _run_pool(net, streams, capacity, "sampling", 77, 5 + capacity)
    _check(got, want, which)
    sizes = [len(g) for c in calls for _, g in c.admit]
    assert len(sizes) >= 3 and max(sizes) < sms // 2, sizes
    assert pool.W == form[1] and pool.CL == form[2]


@pytest.mark.parametrize("park_below,mode", [(1, "argmax"), (80, "sampling")])
def test_parking_pool_equals_one_shot(park_below, mode, monkeypatch):
    cfg, net = _model(BASE30)
    streams = _streams(cfg, 40, 90 + park_below)
    want = _one_shot(net, streams, mode, 5, 16)
    calls = _trace(monkeypatch)
    pool, got = _run_parking_pool(net, streams, 16, mode, 5, 33 + park_below, park_below)
    assert not pool.active and not pool.waiting and not pool.parked
    _check(got, want, (park_below, mode))
    moves = _moves(calls)
    assert len(moves) >= 5 and any(a != b for _, _, _, a, b in moves), moves     # resumed, into other rows too


def test_cancel_and_rebase_with_parked_streams(monkeypatch):
    from pytorchwavenetvocoder_b200.nets import wavenet
    cfg, net = _model(SHALLOW10)
    streams = _streams(cfg, 30, 17)
    want = _one_shot(net, streams, "sampling", 9, 8)
    period = max(cfg.dilations)   # lcm of the queue lengths, and the pool's lowest step
    monkeypatch.setattr(wavenet, "POOL_COUNTER_LIMIT", period + period + 97)
    calls = _trace(monkeypatch)
    cancel_after = {3: 0, 7: 60, 12: 10}
    pool, got = _run_parking_pool(net, streams, 8, "sampling", 9, 21, 8, cancel_after)
    g0s = [c.g0 for c in calls]
    assert min(g0s) >= period and sum(b < a for a, b in zip(g0s, g0s[1:])) >= 3, g0s
    assert _moves(calls)
    for k in range(len(streams)):
        if k in cancel_after:
            assert pool.finished(k) and torch.equal(got[k], want[k][:got[k].numel()]), k
        else:
            assert torch.equal(got[k], want[k]), k


def _rolled(block, rot, qlens, R):
    """torch.roll restatement of wnb_decode_pool_move on one block: each layer's slot range rolled by rot"""
    out, q0 = [], 0
    b = block.view(-1, R)
    for q in qlens:
        out.append(torch.roll(b[q0:q0 + q], rot % q, 0))
        q0 += q
    return torch.cat(out).view(-1)


def test_move_round_trip_and_transplant_are_bit_exact():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import _warp_prefill, ptr, stream
    lib = _lib.load()
    cfg, net = _model(BASE30)
    R, ks, L, capacity = cfg.n_resch, cfg.kernel_size, len(cfg.dilations), 70
    dil = (ctypes.c_int32 * L)(*cfg.dilations)
    qlens = [(ks - 1) * d for d in cfg.dilations]
    block = lib.wnb_decode_workspace(1, R, ks, dil, L) // 4
    g = torch.Generator(device="cuda").manual_seed(5)
    queues = torch.randn(capacity * block, device="cuda", generator=g)
    rows = queues.view(capacity, block)

    def move(src, dst, rot):
        n = len(src)
        _lib.check(lib.wnb_decode_pool_move((ctypes.c_void_p * n)(*src), (ctypes.c_void_p * n)(*dst),
                                            (ctypes.c_int32 * n)(*rot), n, R, ks, dil, L, stream()), "pool_move")

    rng = np.random.RandomState(3)
    for n in (1, 7, 64):
        before = rows.clone()
        src = [int(v) for v in rng.choice(capacity, n, replace=False)]
        dst = [int(v) for v in rng.choice(capacity, n, replace=False)]
        rot = [int(v) for v in rng.randint(-100000, 100000, n)]
        stores = [torch.full((block,), float("nan"), device="cuda") for _ in range(n)]
        move([ptr(rows[s]) for s in src], [ptr(t) for t in stores], rot)
        for i in range(n):
            assert torch.equal(stores[i], _rolled(before[src[i]], rot[i], qlens, R)), (n, i)
        move([ptr(t) for t in stores], [ptr(rows[d]) for d in dst], [-r for r in rot])
        for i in range(n):
            assert torch.equal(rows[dst[i]], before[src[i]]), (n, i)
        untouched = [r for r in range(capacity) if r not in dst]
        assert torch.equal(rows[untouched], before[untouched]), n
    # a transplant from an admission prefill's workspace, as DecodePool admits a group
    w, upw, upb = net._decode_pack(), net.upsampling.conv.weight.detach().reshape(-1).contiguous(), \
        net.upsampling.conv.bias.detach().contiguous()
    Bg, P = 5, cfg.receptive_field + 3
    xs = torch.randint(0, 256, (Bg, P), dtype=torch.int32, device="cuda")
    h = torch.randn(Bg, cfg.n_aux, P // 80 + 2, device="cuda")
    admit = torch.full((Bg * block,), float("nan"), device="cuda")
    _warp_prefill(lib, xs, P, h, upw, upb, w, dil, L, admit, 0, cfg.n_aux, 80, 2)
    dst = [3, 69, 0, 41, 12]
    rot = [1234 - (P - 1), -7, 0, 2 ** 30, -(2 ** 30) - 5]
    move([ptr(admit) + 4 * b * block for b in range(Bg)], [ptr(rows[d]) for d in dst], rot)
    a = admit.view(Bg, block)
    for b in range(Bg):
        assert not torch.isnan(a[b]).any()
        assert torch.equal(rows[dst[b]], _rolled(a[b], rot[b], qlens, R)), b


def test_admission_prefills_at_the_pools_cl(monkeypatch):
    """The queues an admission leaves in a CL 1 pool's rows, un-rotated, equal a CL 1 prefill of the same seed and aux
    bit for bit, and differ from a CL 2 prefill, which is what each group of fewer than sms/2 streams would get on its
    own (wnb_decode_warp_cluster(len(group)) == 2).  Codes alone would rarely show a one-ulp difference in a tap."""
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets import wavenet
    from pytorchwavenetvocoder_b200.nets.wavenet import _decode_snapshot, _warp_prefill
    lib = _lib.load()
    cfg, net = _model(BASE30)
    R, ks, L, A, U = cfg.n_resch, cfg.kernel_size, len(cfg.dilations), cfg.n_aux, cfg.upsampling_factor
    capacity = _sms() // 2 + 1
    assert _form(capacity, L)[2] == 1
    dil = (ctypes.c_int32 * L)(*cfg.dilations)
    qlens = [(ks - 1) * d for d in cfg.dilations]
    block = lib.wnb_decode_workspace(1, R, ks, dil, L) // 4
    snaps = []
    real = wavenet.DecodePool._admit_group

    def traced(self, lib_, T0, group, g0):   # the pool's queues right after the admission, before the decode runs
        real(self, lib_, T0, group, g0)
        snaps.append((T0, [st.sid for st in group], [st.slot for st in group], g0, self.queues.clone()))
    monkeypatch.setattr(wavenet.DecodePool, "_admit_group", traced)
    streams = _streams(cfg, 8, 123, lengths=(20, 41))   # seeds of 1, rf + 2000 and 5 rf + 3: three groups of <= 3
    pool = net.decode_pool(capacity, "sampling", 7)
    for k, (x, total, h, _) in enumerate(streams):
        pool.admit(x, total, h, stream=k)
    pool.step(5)
    assert len(snaps) == 3, [s[:4] for s in snaps]
    w, upw, upb = _decode_snapshot(net)
    for T0, sids, slots, g0, queues in snaps:
        assert lib.wnb_decode_warp_cluster(len(sids)) == 2
        P, Bg = max(T0, cfg.receptive_field), len(sids)
        xs = torch.full((Bg, P), cfg.n_quantize // 2, dtype=torch.int32, device="cuda")   # the padded seed prefix
        xs[:, P - T0:] = torch.stack([streams[k][0].to(torch.int32) for k in sids])
        Fg = min(streams[k][2].size(1) for k in sids)
        h = torch.stack([streams[k][2][:, :Fg] for k in sids]).contiguous()
        ref = {}
        for CL in (1, 2):
            ws = torch.full((Bg * block,), float("nan"), device="cuda")
            _warp_prefill(lib, xs, P, h, upw, upb, w, dil, L, ws, P - T0, A, U, CL)
            ref[CL] = ws.view(Bg, block)
        rows = queues.view(torch.float32).view(capacity, block)
        for i, slot in enumerate(slots):
            got = _rolled(rows[slot], -(g0 - (P - 1)), qlens, R)
            assert torch.equal(got.view(torch.int32), ref[1][i].view(torch.int32)), (T0, i)
            assert not torch.equal(got.view(torch.int32), ref[2][i].view(torch.int32)), (T0, i)


def test_launch_counts():
    """steady call: the inputs kernel and the decode (2); admitting call (one group, L layers): the prefill's front and
    L - 1 layer launches, one move, the inputs kernel and the decode (L + 3); a call that parks one stream and resumes
    another: one move each way and the two (4); a call with nothing to run: none"""
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = _model(SHALLOW10)
    L = len(cfg.dilations)
    pool = net.decode_pool(8, "sampling", 3, park_below=1)
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    h = torch.randn(28, 40, device="cuda")
    pool.admit(x, 1000, h[:, :2])
    pool.admit(x, 1000, h[:, :2])

    def call():
        l0 = _lib.launch_count()
        out = pool.step()
        torch.cuda.synchronize()
        return _lib.launch_count() - l0, sorted(out)

    assert call() == (L + 3, [0, 1])          # 2 frames of U 80: samples 0 .. 159
    assert call() == (0, [])
    pool.feed(1, h[:, 2:4])
    assert call() == (3, [1]) and pool.parked == [0]
    pool.feed(0, h[:, 2:4])
    assert call() == (4, [0]) and pool.parked == [1]
    pool.feed(0, h[:, 4:6])
    pool.feed(1, h[:, 4:6])
    pool.step()                               # resumes 1
    pool.feed(0, h[:, 6:8])
    pool.feed(1, h[:, 6:8])
    assert call() == (2, [0, 1])


def test_step_pcm16_equals_codes():
    from pytorchwavenetvocoder_b200.nets.wavenet import codes_to_pcm16
    cfg, net = _model(SHALLOW10)
    streams = _streams(cfg, 3, 5)
    want = _one_shot(net, streams, "sampling", 4, 4)
    pool = net.decode_pool(4, "sampling", 4)
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
    with pytest.raises(_lib.WnbError, match="warp decoder"):
        WaveNet(256, 28, 256, 256, 3, 1, 2, 4).cuda().decode_pool(8)      # 256/256 under fp32
    with pytest.raises(_lib.WnbError, match="warp decoder"):
        WaveNet(256, 28, 64, 512, 3, 1, 3, 4).cuda().decode_pool(8)       # ks 3
    _, net = _model(SHALLOW10)
    with pytest.raises(ValueError):
        net.decode_pool(0)


# ---- bin/decode.py --pool_capacity ---------------------------------------------------------------------------------
def _cli(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.decode"] + args, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    assert r.returncode == 0, r.stdout.decode()[-3000:]


@pytest.mark.parametrize("gpus", [1, 2])
@pytest.mark.parametrize("math", ["fp32", "bf16"])
def test_cli_pool_writes_the_pool_api_files(tmp_path, math, gpus):
    """decode.py --pool_capacity 8 writes the wavs of a direct pool run with the worker's drawn seed, with and without
    --noise_shaping (then: mlsa_filter_batch of the pool's PCM_16)"""
    from pytorchwavenetvocoder_b200.bin import decode as D
    from pytorchwavenetvocoder_b200.nets import WaveNet, codes_to_pcm16, decode_mu_law
    from pytorchwavenetvocoder_b200.utils import have_soundfile, write_hdf5, write_wav, write_wav_pcm16
    from pytorchwavenetvocoder_b200.utils.mlsa import convert_mcep_to_mlsa_coef, mlsa_filter_batch
    if gpus > torch.cuda.device_count():
        pytest.skip("needs %d GPUs" % gpus)
    U, D_ = 16, 28
    R, S, depth = (64, 512, 4) if math == "fp32" else (256, 256, 3)
    rng = np.random.RandomState(12)
    torch.manual_seed(0)
    net = WaveNet(256, D_, R, S, depth, 2, 2, U)
    expdir, featdir = tmp_path / "exp", tmp_path / "feats"
    expdir.mkdir()
    featdir.mkdir()
    ckpt = str(expdir / "checkpoint-final.pkl")
    torch.save({"model": net.state_dict()}, ckpt)
    conf = argparse.Namespace(n_quantize=256, n_aux=D_, n_resch=R, n_skipch=S, dilation_depth=depth, dilation_repeat=2,
                              kernel_size=2, upsampling_factor=U, use_upsampling_layer=True, feature_type="world",
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
              str(gpus), "--decode_math", math, "--pool_capacity", "8", "--batch_size", "3"]
    plain, shaped = str(tmp_path / "plain"), str(tmp_path / "shaped")
    _cli(common + ["--outdir", plain])
    _cli(common + ["--outdir", shaped, "--noise_shaping"])
    # the direct pool run of every worker: stream id = index in the worker's list, seed = pool_seed(5, gpu)
    net = net.cuda().eval()
    net.decode_math = math
    scaler = D.load_scaler(stats, "world")
    for gpu, idx in enumerate(np.array_split(np.arange(len(feats)), gpus)):
        seed = D.pool_seed(5, gpu)
        with torch.no_grad():
            pool = net.decode_pool(8, "sampling", seed)
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
            assert open(os.path.join(plain, name), "rb").read() == open(want, "rb").read(), (math, gpus, i)
            pcm = codes_to_pcm16(codes, 256).cpu().numpy()
            write_wav_pcm16(want, mlsa_filter_batch([pcm], coef, 0.41, 4)[0], 16000)
            assert open(os.path.join(shaped, name), "rb").read() == open(want, "rb").read(), (math, gpus, i)
