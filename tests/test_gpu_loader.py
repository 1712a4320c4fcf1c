# -*- coding: utf-8 -*-
"""GPU tier (SURVEY.md 8f-1): the on-device train_generator (utils/device_loader.py + csrc/loader.cu) yields exactly the
batches of the host generator (bin/train.py train_generator = reference train.py:67-312) on the same file lists, also
after its device rings have wrapped; and wnb_make_train_batch alone equals the numpy restatement of
tests/loader_reference.py bit for bit at the rings' edges, in every scaler mode."""
import os

import numpy as np
import pytest
import torch

from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["float64", "float32"])
def corpus(request, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("corpus_" + request.param))
    rng = np.random.RandomState(0)
    U, D = 80, 28
    wavs, feats = [], []
    for i, n_frames in enumerate([90, 120, 75, 101, 33, 140]):
        n = n_frames * U + rng.randint(-30, 30)
        w = os.path.join(root, "u%d.wav" % i)
        f = os.path.join(root, "u%d.npz" % i)
        write_wav(w, 0.6 * np.sin(np.arange(n) / (7.0 + i)) * np.cos(np.arange(n) / 301.0), 16000)
        feat = rng.standard_normal((n_frames, D))
        write_hdf5(f, "/world", feat.astype(request.param))     # both storage dtypes the recipes produce
        write_hdf5(f, "/speaker_code", np.eye(3)[i % 3].astype(request.param))
        wavs.append(w)
        feats.append(f)
    mean = rng.standard_normal(D + 3)
    scale = 0.5 + rng.rand(D + 3)
    return wavs, feats, U, D, mean, scale


@pytest.mark.parametrize("batch_length,batch_size,use_up,shuffle,use_spk", [
    (2000, 3, True, False, False), (1500, 2, False, False, False), (2000, 4, True, True, False), (900, 1, True, False, False),
    (2000, 2, True, False, True), (1200, 2, False, True, True)])      # use_speaker_code: reference train.py:123-128
def test_device_generator_matches_host_generator(corpus, batch_length, batch_size, use_up, shuffle, use_spk):
    from sklearn.preprocessing import StandardScaler
    from pytorchwavenetvocoder_b200.bin.train import train_generator
    from pytorchwavenetvocoder_b200.nets import encode_mu_law
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceTrainGenerator
    wavs, feats, U, D, mean, scale = corpus
    if not use_spk:
        mean, scale = mean[:D], scale[:D]
    rf = 1 + 1023
    scaler = StandardScaler()
    scaler.mean_, scaler.scale_ = mean, scale
    np.random.seed(5)
    host = train_generator(wavs, feats, receptive_field=rf, batch_length=batch_length, batch_size=batch_size,
                           wav_transform=lambda x: encode_mu_law(x, 256), feat_transform=scaler.transform,
                           shuffle=shuffle, upsampling_factor=U, use_upsampling_layer=use_up, use_speaker_code=use_spk)
    want = [host.next() for _ in range(12)]          # > 1 epoch of this corpus: crosses the reshuffle
    np.random.seed(5)
    devg = DeviceTrainGenerator(wavs, feats, rf, batch_length, batch_size, n_quantize=256, mean=mean, scale=scale,
                                shuffle=shuffle, upsampling_factor=U, use_upsampling_layer=use_up,
                                use_speaker_code=use_spk)
    for k, ((xw, hw), tw) in enumerate(want):
        (x, h), t = devg.next()
        assert x.is_cuda and x.dtype == torch.int64 and h.dtype == torch.float32
        assert torch.equal(x.cpu(), xw.cpu()), k
        assert torch.equal(t.cpu(), tw.cpu()), k
        assert h.size(1) == D + (3 if use_spk else 0)
        assert torch.equal(h.cpu(), hw.cpu()), (k, (h.cpu() - hw.cpu()).abs().max())


# ------------------------------------------------------------------------------------------------------------------
# wnb_make_train_batch called directly, against the numpy restatement of tests/loader_reference.py, bit for bit
# ------------------------------------------------------------------------------------------------------------------
from tests import loader_reference as R                      # noqa: E402
from tests.test_gpu_tc_stages import PAD, Guarded           # noqa: E402

POISON_I64 = -(1 << 40)                                      # never a mu-law code
SENTINEL_I64 = 0x5A5A5A5A5A5A5A5A


class GuardedI64(Guarded):
    """int64 outputs as slices of sentinel-filled buffers"""

    def __call__(self, shape, fill=POISON_I64):
        n = int(np.prod(shape))
        buf = torch.full((n + 2 * PAD,), SENTINEL_I64, dtype=torch.int64, device="cuda")
        v = buf[PAD:PAD + n].view(*shape)
        v.fill_(fill)
        self.bufs.append(buf)
        return v

    def check(self):
        for i, b in enumerate(self.bufs):
            assert torch.all(b[:PAD] == SENTINEL_I64) and torch.all(b[-PAD:] == SENTINEL_I64), "write outside output %d" % i


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid_x(T, Tf, D):
    work = max(T + 1, D * Tf)
    return min(-(-work // 256), _sms())


def _launch(wave, feat, fos, s0, hop, U, cap_s, cap_f, mean, scale, x, t, h, B, T, Tf, D, feat_f64, mu):
    from pytorchwavenetvocoder_b200 import _lib
    P = _lib.ptr
    _lib.check(_lib.load().wnb_make_train_batch(P(wave), P(feat), P(fos), s0, hop, U, cap_s, cap_f, P(mean), P(scale),
                                                P(x), P(t), P(h), B, T, Tf, D, feat_f64, mu, _lib.stream()),
               "make_train_batch")


def _run_case(c, mode, wave32, mu=256, seed=0):
    """one launch of geometry c in scaler mode `mode` on the wave ring wave32; compares x, t, h bit for bit with the
    restatement (codes of the ring's samples from nets.encode_mu_law, the elementwise.cu twin of the loader's mu-law)"""
    from pytorchwavenetvocoder_b200.nets import encode_mu_law
    dt, feat_f64, with_scaler = R.scaler_mode_args(mode)
    rng = np.random.RandomState(seed)
    D, B, T, Tf = c["D"], c["B"], c["T"], c["Tf"]
    feat = (rng.standard_normal((c["cap_f"], D)) * 10.0 ** rng.uniform(-2, 2, (c["cap_f"], D))).astype(dt)
    mean = rng.standard_normal(D) * 2 if with_scaler else None
    scale = 0.1 + rng.rand(D) * 3 if with_scaler else None
    fos = R.fos_ring(c) if c["fos"] else None
    g, gi = Guarded(), GuardedI64()
    x, t = gi((B, T)), gi((B, T))
    h = g((B, D, Tf))
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    _launch(dev(wave32), dev(feat), dev(fos), c["s0"], c["hop"], c["U"], c["cap_s"], c["cap_f"], dev(mean), dev(scale),
            x, t, h, B, T, Tf, D, feat_f64, mu)
    torch.cuda.synchronize()
    g.check()
    gi.check()
    codes = encode_mu_law(wave32, mu)
    xw, tw, hw = R.make_train_batch(codes, feat, fos, c["s0"], c["hop"], c["U"], c["cap_s"], c["cap_f"], mean, scale,
                                    B, T, Tf, mode)
    for name, got, want in (("x", x, xw), ("t", t, tw), ("h", h, hw)):
        got = got.cpu().numpy()
        bad = np.argwhere(got != want) if name != "h" else np.argwhere(~(got == want))
        assert bad.size == 0, "%s differs at %d elements, first (row, ...) %s: got %r want %r (so %% cap_s = %d)" % (
            name, len(bad), tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])],
            (c["s0"] + int(bad[0][0]) * c["hop"]) % c["cap_s"])
    return codes, x, t


def _wave(n, seed):
    rng = np.random.RandomState(seed)
    return (rng.randint(-32768, 32768, n) / 32768.0).astype(np.float32)


@pytest.mark.parametrize("mode", R.SCALER_MODES)
@pytest.mark.parametrize("name", sorted(R.RING_CASES))
def test_make_train_batch_ring_edges_bit_exact(name, mode):
    """windows ending at cap_s - 1 and at cap_s, straddling the ring end at several offsets, cap_s = T + 1, a feature
    ring wrapping at another window, hop = 0, s0 >= 2^32; in every scaler mode"""
    c = R.ring_case(name)
    print("scaler mode %s, case %s: %s" % (mode, name, ", ".join(sorted(set(c["reaches"])))))
    _run_case(c, mode, _wave(c["cap_s"], 3))


@pytest.mark.parametrize("mu", [256, 1024])
def test_make_train_batch_mulaw_domain(mu):
    """a wave ring holding every PCM-16 value, the quantiser's near-edge floats and +-1, +-0, with cap_s = T + 1 so one row
    reads every slot: codes equal nets.encode_mu_law everywhere, the float64-log restatement everywhere, and the numpy
    oracle outside the edge mask"""
    from oracle.wavenet_oracle import encode_mu_law as oracle_enc
    from tests.golden.cases import mulaw_pcm16_domain
    vals = np.concatenate([mulaw_pcm16_domain(), R.mulaw_near_edges(mu), np.float32([1, -1, 0, -0.0])])
    U = 80
    T = -(-len(vals) // U) * U
    cap_s = T + 1
    wave = np.concatenate([vals, _wave(cap_s - len(vals), 4)]).astype(np.float32)
    wave = wave[np.random.RandomState(mu).permutation(cap_s)]
    c = dict(fos=False, U=U, T=T, Tf=T // U, D=4, B=2, hop=U * 7, cap_s=cap_s, cap_f=T // U + 3, s0=U * 1001)
    codes, x, t = _run_case(c, "f32_none", wave, mu=mu)
    # row 0 reads every slot: x holds slots so .. so + T - 1, t the slot after the last
    got = np.empty(cap_s, np.int64)
    so = c["s0"] % cap_s
    got[(so + np.arange(T)) % cap_s] = x[0].cpu().numpy()
    got[(so + T) % cap_s] = t[0, -1].item()
    assert np.array_equal(got, codes)
    ref = R.mulaw_f32_reference(wave, mu)
    assert np.array_equal(got, ref), np.nonzero(got != ref)
    o = oracle_enc(wave, mu)
    mask = R.mulaw_edge_mask_mu(wave, mu)
    assert not np.any((got != o) & ~mask), wave[(got != o) & ~mask]
    assert got.min() == 0 and got.max() == mu - 1
    print("mu %d: %d slots, %d within 2 ulp of an edge, %d of those differ from numpy" % (
        mu, cap_s, int(mask.sum()), int(((got != o) & mask).sum())))


def _shape_cases():
    S = _sms()
    Tf_big = -(-256 * S // 28) + 7           # D * Tf > 256 * SMs at D = 28
    return {
        # T + 1 dominates (up-sampling, Tf = T / U), B = 1
        "up_T_dominates_B1": dict(fos=False, U=80, T=4000, D=28, B=1, hop=0, cap_s=4500, cap_f=60, s0=80 * 50),
        # D * Tf dominates (frame_of_sample, Tf = T), rows that share nothing
        "fos_DTf_dominates_B24": dict(fos=True, U=80, T=1000, D=28, B=24, hop=1100, cap_s=26501, cap_f=1100, s0=12345),
        # both grid-stride loops run more than once: T + 1 > 256 * SMs and D * Tf > 256 * SMs
        "up_multi_pass": dict(fos=False, U=80, T=Tf_big * 80, D=28, B=2, hop=80 * 37, cap_s=Tf_big * 80 + 4001,
                              cap_f=Tf_big + 11, s0=80 * 999),
        "fos_multi_pass": dict(fos=True, U=80, T=256 * S + 300, D=28, B=3, hop=5000, cap_s=256 * S + 7000,
                               cap_f=256 * S + 310, s0=(256 * S + 7000) * 2 - 100),
    }


@pytest.mark.parametrize("name", ["up_T_dominates_B1", "fos_DTf_dominates_B24", "up_multi_pass", "fos_multi_pass"])
def test_make_train_batch_launch_shapes(name):
    """the grid is min(cdiv(max(T + 1, D * Tf), 256), SMs) x B: cases where either loop sets it, and where the work exceeds
    256 * SMs so each grid-stride loop runs more than once"""
    c = _shape_cases()[name]
    c["Tf"] = c["T"] if c["fos"] else c["T"] // c["U"]
    gx = _grid_x(c["T"], c["Tf"], c["D"])
    passes = (-(-(c["T"] + 1) // (gx * 256)), -(-(c["D"] * c["Tf"]) // (gx * 256)))
    print("case %s: grid %d x %d, grid-stride passes (wave, features) %s" % (name, gx, c["B"], passes))
    if "T_dominates" in name:
        assert c["T"] + 1 > c["D"] * c["Tf"] and c["B"] == 1
    if "DTf_dominates" in name:
        assert c["D"] * c["Tf"] > c["T"] + 1 and c["B"] * c["hop"] > c["T"]
    if "multi_pass" in name:
        assert min(passes) > 1
    for mode in ("mode0", "f64"):
        _run_case(c, mode, _wave(c["cap_s"], 5))


@pytest.mark.parametrize("bad", ["cap_s_eq_T", "cap_s_lt_T", "cap_f_lt_Tf", "mean_without_scale", "scale_without_mean",
                                 "mu_1", "s0_negative", "B_0"])
def test_make_train_batch_rejects_bad_arguments(bad):
    from pytorchwavenetvocoder_b200 import _lib
    c = dict(U=80, T=800, Tf=10, D=28, B=2, hop=80, cap_s=1000, cap_f=12, s0=160, mu=256)
    rng = np.random.RandomState(0)
    wave = torch.from_numpy(_wave(1000, 1)).cuda()
    feat = torch.from_numpy(rng.standard_normal((12, 28)).astype(np.float32)).cuda()
    mean = torch.zeros(28, dtype=torch.float64, device="cuda")
    scale = torch.ones(28, dtype=torch.float64, device="cuda")
    mean_, scale_ = mean, scale
    if bad == "cap_s_eq_T":
        c["cap_s"] = c["T"]
    elif bad == "cap_s_lt_T":
        c["cap_s"] = c["T"] - 1
    elif bad == "cap_f_lt_Tf":
        c["cap_f"] = c["Tf"] - 1
    elif bad == "mean_without_scale":
        scale_ = None
    elif bad == "scale_without_mean":
        mean_ = None
    elif bad == "mu_1":
        c["mu"] = 1
    elif bad == "s0_negative":
        c["s0"] = -80
    elif bad == "B_0":
        c["B"] = 0
    g, gi = Guarded(), GuardedI64()
    x, t, h = gi((2, 800)), gi((2, 800)), g((2, 28, 10))
    with pytest.raises(_lib.WnbError, match="bad arguments"):
        _launch(wave, feat, None, c["s0"], c["hop"], c["U"], c["cap_s"], c["cap_f"], mean_, scale_, x, t, h, c["B"],
                c["T"], c["Tf"], c["D"], 2, c["mu"])
    torch.cuda.synchronize()
    g.check()
    gi.check()
    assert torch.all(x == POISON_I64) and torch.all(t == POISON_I64) and torch.all(torch.isnan(h))
    # cap_s = T + 1 is the smallest accepted capacity
    if bad == "cap_s_eq_T":
        _run_case(dict(fos=False, U=80, T=800, Tf=10, D=28, B=2, hop=80, cap_s=801, cap_f=10, s0=160), "mode2",
                  _wave(801, 2))


# ------------------------------------------------------------------------------------------------------------------
# DeviceTrainGenerator through real wraparound of its rings, against bin.train.train_generator
# ------------------------------------------------------------------------------------------------------------------
WRAP_U, WRAP_D, WRAP_RF = 80, 28, 1 + 1023

WRAP_CASES = {
    # the training defaults (--batch_length 20000 --batch_size 1): capacity 1 << 22
    "up_f32_default": dict(batch_length=20000, batch_size=1, use_up=True, ftype="world", spk=False),
    "up_f64_speaker": dict(batch_length=12000, batch_size=3, use_up=True, ftype="melspc", spk=True),
    "extend_time_f32": dict(batch_length=15000, batch_size=2, use_up=False, ftype="world", spk=False),
    "extend_time_f64": dict(batch_length=9000, batch_size=4, use_up=False, ftype="melspc", spk=False),
    # T + 2 + hop * B * 6 > 1 << 22: a capacity that is not a power of two, and cap_f * U != cap_s
    "up_f32_big_ring": dict(batch_length=20000, batch_size=40, use_up=True, ftype="world", spk=False),
}


@pytest.fixture(scope="module")
def wrap_corpus(tmp_path_factory):
    """40 utterances of 1.5-6 s at 16 kHz (U = 80, none a multiple of U), features as float32 (/world) and float64
    (/melspc), speaker codes"""
    root = str(tmp_path_factory.mktemp("wrap_corpus"))
    rng = np.random.RandomState(11)
    U, D = WRAP_U, WRAP_D
    wavs, feats = [], []
    for i in range(40):
        n_frames = rng.randint(300, 1201)
        n = n_frames * U + rng.choice([-1, 1]) * rng.randint(1, U)
        assert n % U != 0
        k = np.arange(n)
        w = 0.5 * np.sin(k / (5.0 + i)) * np.cos(k / (411.0 + 7 * i)) + 0.05 * rng.standard_normal(n)
        wp, fp = os.path.join(root, "w%02d.wav" % i), os.path.join(root, "w%02d.npz" % i)
        write_wav(wp, np.clip(w, -0.99, 0.99), 16000)
        f = rng.standard_normal((n_frames, D)) * 10.0 ** rng.uniform(-1, 1, D)
        write_hdf5(fp, "/world", f.astype(np.float32))
        write_hdf5(fp, "/melspc", f[::-1].copy())
        write_hdf5(fp, "/speaker_code", np.eye(3)[i % 3].astype(np.float32))
        wavs.append(wp)
        feats.append(fp)
    mean = rng.standard_normal(D + 3)
    scale = 0.5 + rng.rand(D + 3)
    return wavs, feats, mean, scale


def _utterance_order(wavs, feats, epochs, seed):
    """the file pairs both generators visit: one permutation of the current lists per epoch from a RNG seeded `seed`"""
    rs = np.random.RandomState(seed)
    wl, fl, order = list(wavs), list(feats), []
    for _ in range(epochs):
        idx = rs.permutation(len(wl))
        wl, fl = [wl[i] for i in idx], [fl[i] for i in idx]
        order.extend((w, f, i + 1 == len(wl)) for i, (w, f) in enumerate(zip(wl, fl)))
    return order


@pytest.mark.parametrize("name", list(WRAP_CASES))
def test_device_generator_through_ring_wraparound(wrap_corpus, name):
    """stream > 2.5 rings' worth of samples (several shuffled epochs) through DeviceTrainGenerator and compare every
    batch with the host generator; the windows, replayed with WindowPlanner over the same utterance lengths, must include
    ones that straddle the end of the sample ring and of the feature ring, and slots must have been overwritten"""
    from sklearn.preprocessing import StandardScaler
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.bin.train import train_generator
    from pytorchwavenetvocoder_b200.nets import encode_mu_law
    from pytorchwavenetvocoder_b200.utils.device_loader import DeviceTrainGenerator, WindowPlanner, load_pair_frames
    c = WRAP_CASES[name]
    wavs, feats, mean, scale = wrap_corpus
    U, B = WRAP_U, c["batch_size"]
    if not c["spk"]:
        mean, scale = mean[:WRAP_D], scale[:WRAP_D]
    lengths = {}
    for w, f in zip(wavs, feats):
        x_, h_ = load_pair_frames(w, f, c["ftype"], U, c["use_up"], False)
        lengths[w] = (len(x_), len(h_))
    epoch_samples = sum(n for n, _ in lengths.values())

    np.random.seed(5)
    devg = DeviceTrainGenerator(wavs, feats, WRAP_RF, c["batch_length"], B, feature_type=c["ftype"], n_quantize=256,
                                mean=mean, scale=scale, shuffle=True, upsampling_factor=U,
                                use_upsampling_layer=c["use_up"], use_speaker_code=c["spk"])
    T, Tf, hop, cap_s = devg.T, devg.Tf, devg.hop, devg.cap_s
    target = int(2.5 * cap_s)
    epochs = -(-(target + B * hop + T) // epoch_samples) + 3
    # plan every epoch the test can reach now, so the device generator's reader threads draw no permutation while the
    # host generator draws the same sequence from the re-seeded global RNG
    devg._utterance(epochs * len(wavs) - 1)
    order = _utterance_order(wavs, feats, epochs, 5)
    assert [o[:2] for o in devg._order[:len(order)]] == [o[:2] for o in order]
    np.random.seed(5)
    scaler = StandardScaler()
    scaler.mean_, scaler.scale_ = mean, scale
    host = train_generator(wavs, feats, receptive_field=WRAP_RF, batch_length=c["batch_length"], batch_size=B,
                           feature_type=c["ftype"], wav_transform=lambda x: encode_mu_law(x, 256),
                           feat_transform=scaler.transform, shuffle=True, upsampling_factor=U,
                           use_upsampling_layer=c["use_up"], use_speaker_code=c["spk"])

    # window starts and frame positions, replayed on the utterance lengths
    plan = WindowPlanner(B, hop, devg.need)
    starts_s, starts_f, pos_s, pos_f = [], [], 0, 0
    for w, _, last in order:
        n, nf = lengths[w]
        starts_s.append(pos_s)
        starts_f.append(pos_f)
        pos_s += n
        pos_f += nf
        plan.append(n, last)
    starts_s, starts_f = np.array(starts_s), np.array(starts_f)
    n_batches = next(k for k, s0 in enumerate(plan.ready) if s0 >= target) + 1

    def frame(p):
        u = np.searchsorted(starts_s, p, side="right") - 1
        return int(starts_f[u] + (p - starts_s[u]) // U)

    cap_f = devg.cap_f
    straddle_s = straddle_f = 0
    for k in range(n_batches):
        try:
            (x, h), t = devg.next()
        except _lib.WnbError as e:
            pytest.fail("batch %d: %s" % (k, e))
        (xw, hw), tw = host.next()
        s0 = plan.ready[k]
        where = "batch %d (s0 %d, ring slot %d of %d)" % (k, s0, s0 % cap_s, cap_s)
        assert torch.equal(x, xw), "x " + where
        assert torch.equal(t, tw), "t " + where
        assert torch.equal(h, hw), "h " + where
        for b in range(B):
            so = s0 + b * hop
            straddle_s += so % cap_s + T >= cap_s
            f_first = frame(so)
            f_last = f_first + Tf - 1 if c["use_up"] else frame(so + T - 1)
            straddle_f += f_first // cap_f != f_last // cap_f
    print("case %s: cap_s %d, cap_f %d, T %d, hop %d, B %d, %d batches: sample ring wrapped %d times, feature ring %d "
          "times; %d windows straddle the end of the sample ring, %d of the feature ring" % (
              name, cap_s, cap_f, T, hop, B, n_batches, devg.tail_s // cap_s, devg.tail_f // cap_f, straddle_s,
              straddle_f))
    assert devg.tail_s > 2 * cap_s                   # slots overwritten twice over were read
    assert straddle_s >= 1 and straddle_f >= 1
    if name == "up_f32_default":
        assert cap_s == 1 << 22
    if name == "up_f32_big_ring":
        assert cap_s > 1 << 22 and cap_s & (cap_s - 1) and cap_f * U != cap_s
