# -*- coding: utf-8 -*-
"""CPU tier of held-out scoring (utils/scoring.py, bin/evaluate.py, train.py --dev_*): the window plan by brute force,
a float64 restatement of wnb_cross_entropy_rows checked against planted mistakes, the utterance alignment against
train_generator, the CLI refusals, the ordered gather under gloo, and the kernel's ptxas counts."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pytorchwavenetvocoder_b200.utils import scoring as S
from tests.score_reference import rows_ce

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the window plan ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("U", [0, 80, 256])
@pytest.mark.parametrize("rf", [2, 5, 64, 97])
def test_window_plan_covers_every_position_once(U, rf):
    unit = S.window_unit(U)
    C = S.window_context(rf, U)
    assert C % unit == 0 and rf - 1 <= C < rf - 1 + unit
    for L in (unit, 2 * unit, 5 * unit):
        for T in range(1, 4 * rf + 1):
            for start in sorted({0, 1, rf - 1, rf, rf + 1, T - 1, T}):
                if start < 0:
                    continue
                hits = np.zeros(T, dtype=np.int64)
                for k, a, s, e in S.score_window_plan(T, rf, U, L, start):
                    assert a % unit == 0 and a <= s < e <= T
                    assert s == start or s % unit == 0                       # interior starts on whole segments/frames
                    assert e - a <= C + L                                      # at most C + L inputs
                    assert a == 0 or s - a >= rf - 1                           # no zero padding the whole lacks
                    if U > 0:
                        assert (e - a) % U == 0 or e == T                        # whole frames
                    hits[s:e] += 1
                assert (hits[start:] == 1).all() and (hits[:start] == 0).all(), (T, start, L)


def test_window_plan_refusals():
    with pytest.raises(ValueError):
        S.score_window_plan(100, 10, 80, 100, 10)       # hop not a multiple of lcm(80, 32)
    with pytest.raises(ValueError):
        S.score_window_plan(100, 10, 0, 0, 10)
    with pytest.raises(ValueError):
        S.score_window_plan(100, 10, 0, 32, -1)
    assert S.window_unit(80) == 160 and S.window_unit(256) == 256 and S.window_unit(0) == 32


def test_score_batches_budget():
    rng = np.random.RandomState(0)
    lengths = list(rng.randint(1, 5000, size=40)) + [9000]
    batches = S.score_batches(lengths, 8000)
    assert sorted(i for b in batches for i in b) == list(range(len(lengths)))
    for b in batches:
        assert all(lengths[b[0]] >= lengths[i] for i in b)
        assert len(b) == 1 or len(b) * lengths[b[0]] <= 8000
    assert [40] in batches                            # longer than the budget: alone


# ---- float64 restatement of the per-row cross entropy --------------------------------------------------------------
def _case(seed=0, B=4, T=50, Q=16):
    rng = np.random.RandomState(seed)
    logits = rng.standard_normal((B, T, Q)).astype(np.float32) * 3
    target = rng.randint(0, Q, size=(B, T)).astype(np.int64)
    lengths = np.array([T, 3, 0, 37][:B], dtype=np.int64)
    return logits, target, lengths


def test_rows_ce_restatement_catches_planted_mistakes():
    logits, target, lengths = _case()
    start = 5
    nll, cnt = rows_ce(logits, target, lengths, start)
    # the restatement itself, against a direct per-position loop
    for b in range(4):
        want = 0.0
        for p in range(start, min(lengths[b], 50)):
            z = logits[b, p].astype(np.float64)
            want += np.log(np.exp(z - z.max()).sum()) + z.max() - z[target[b, p]]
        assert abs(nll[b] - want) <= 1e-12 * max(1.0, abs(want))
    assert list(cnt) == [45, 0, 0, 32] and nll[1] == 0.0 and nll[2] == 0.0
    # an off-by-one start, a wrong target shift and summing the padding all change the answer
    off, _ = rows_ce(logits, target, lengths, start - 1)
    shifted, _ = rows_ce(logits, np.roll(target, 1, axis=1), lengths, start)
    padded, _ = rows_ce(logits, target, np.full(4, 50), start)
    for bad in (off, shifted, padded):
        assert not np.allclose(bad, nll, rtol=1e-9, atol=0)


class _FakeNet(torch.nn.Module):
    """A causal stand-in for WaveNet on the CPU: the logits of position p depend on x[p], x[p - 1] and the aux column of
    p only, so every window of utils.scoring sees what the whole utterance sees.  ``score`` runs the float64
    restatement on those logits; ``mistake`` plants an error in the bookkeeping the host code does around it."""

    def __init__(self, U, rf=6, n_aux=3, Q=16, mistake=None):
        super().__init__()
        self.upsampling_factor, self.receptive_field, self.n_aux, self.n_quantize = U, rf, n_aux, Q
        self.w = torch.nn.Parameter(torch.zeros(1))
        rng = np.random.RandomState(3)
        self.table = rng.standard_normal((Q, Q)) * 2
        self.mix = rng.standard_normal((n_aux, Q))
        self.mistake = mistake

    def logits(self, x, h):
        x, h = np.asarray(x), np.asarray(h, dtype=np.float64)
        U = self.upsampling_factor
        cols = np.repeat(h, U, axis=-1) if U > 0 else h
        prev = np.concatenate([np.zeros_like(x[..., :1]), x[..., :-1]], -1)
        return self.table[x % self.n_quantize] + 0.5 * self.table[prev % self.n_quantize][..., ::-1] + \
            np.einsum("...at,aq->...tq", cols, self.mix)

    def score(self, x, h, t, lengths, start=None, out=None):
        start = self.receptive_field if start is None else start
        lengths = lengths.numpy() if torch.is_tensor(lengths) else np.asarray(lengths)
        t = t.numpy() % self.n_quantize
        if self.mistake == "start":
            start -= 1
        if self.mistake == "shift":
            t = np.roll(t, 1, axis=1)
        if self.mistake == "padding":
            lengths = np.full_like(lengths, x.shape[1])
        nll, cnt = rows_ce(self.logits(x.numpy(), h.numpy()), t, lengths, start)
        if out is None:
            return torch.from_numpy(nll), torch.from_numpy(cnt)
        out[0].add_(torch.from_numpy(nll))
        out[1].add_(torch.from_numpy(cnt))
        return out


@pytest.mark.parametrize("U", [0, 4])
def test_score_utterances_against_the_restatement(U):
    """score_utterances, whole and windowed, against rows_ce of each utterance alone; the planted mistakes (an
    off-by-one start, a wrong target shift, summing the padding) run through the same host code and are caught."""
    rng = np.random.RandomState(5)
    good = _FakeNet(U)
    Ts = [(n // max(U, 1)) * max(U, 1) for n in (700, 95, 5, 6, 7, 333, 64)]   # some no longer than rf
    utts = []
    for T in Ts:
        codes = rng.randint(0, 16, size=T + 1).astype(np.int64)
        utts.append((codes[:T], codes[1:], rng.standard_normal((3, T // U if U else T)).astype(np.float32)))
    want = np.zeros(len(utts)), np.zeros(len(utts), dtype=np.int64)
    for i, (x, t, h) in enumerate(utts):
        n, c = rows_ce(good.logits(x[None], h[None]), t[None], [len(x)], good.receptive_field)
        want[0][i], want[1][i] = n[0], c[0]
    assert list(want[1]) == [max(T - 6, 0) for T in Ts]
    for budget in (1 << 20, 2000, 250):   # 250: the longest utterances are scored in windows
        nll, cnt = S.score_utterances(good, utts, budget)
        assert np.array_equal(cnt, want[1]), budget
        assert np.allclose(nll, want[0], rtol=1e-12, atol=0), budget
        for mistake in ("start", "shift", "padding"):
            bad, _ = S.score_utterances(_FakeNet(U, mistake=mistake), utts, budget)
            assert not np.allclose(bad, want[0], rtol=1e-9, atol=0), (budget, mistake)


# ---- alignment with the training batches ----------------------------------------------------------------------------
def _enc(x, mu=256):   # CPU stand-in for the device mu-law
    from oracle.wavenet_oracle import encode_mu_law
    return encode_mu_law(x, mu)


@pytest.mark.parametrize("U", [0, 80])
def test_utterance_arrays_match_train_generator(tmp_path, U):
    from pytorchwavenetvocoder_b200.bin.train import _load_pair, train_generator
    from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav
    rng = np.random.RandomState(1)
    w, f = str(tmp_path / "u.wav"), str(tmp_path / "u.npz")
    write_wav(w, 0.3 * np.sin(np.arange(80 * 40 + 17) / 9.0), 16000)
    write_hdf5(f, "/world", rng.standard_normal((40, 6)))
    gen = train_generator([w], [f], receptive_field=9, batch_length=None, batch_size=1, wav_transform=_enc,
                          feat_transform=None, shuffle=False, upsampling_factor=80, use_upsampling_layer=U > 0)
    (x, h), t = gen.next()
    xw, hw = _load_pair(w, f, "world", 80, U > 0, False)
    xi, ti, hi = S.utterance_arrays(xw, hw, 256, U, mulaw=_enc)
    assert np.array_equal(xi, x[0].numpy()) and np.array_equal(ti, t[0].numpy())
    assert np.array_equal(hi, h[0].numpy())
    if U > 0:
        assert len(xi) == (len(xw) - 1) // 80 * 80 and hi.shape[1] == len(xi) // 80


def test_utterance_arrays_short():
    xi, ti, hi = S.utterance_arrays(np.zeros(50), np.zeros((1, 3)), 256, 80, mulaw=_enc)
    assert len(xi) == len(ti) == 0 and hi.shape == (3, 0)


def test_corpus_mean_skips_empty_and_is_never_nan_per_utterance():
    s, n, mean = S.corpus_mean([1.5, 0.0, 2.25], [3, 0, 4])
    assert (s, n) == (3.75, 7) and mean == 3.75 / 7
    assert np.isnan(S.corpus_mean([0.0], [0])[2])


# ---- CLI refusals ---------------------------------------------------------------------------------------------------
def test_evaluate_refusals(tmp_path):
    from pytorchwavenetvocoder_b200.bin import evaluate as E
    from pytorchwavenetvocoder_b200.utils import write_hdf5
    a, b = tmp_path / "w.scp", tmp_path / "f.scp"
    a.write_text("x1.wav\nx2.wav\n")
    b.write_text("x1.h5\n")
    with pytest.raises(ValueError, match="2 waveforms but 1"):
        E.file_lists(str(a), str(b))
    with pytest.raises(ValueError):
        E.file_lists(str(tmp_path / "missing"), str(b))
    stats = str(tmp_path / "stats.npz")
    write_hdf5(stats, "/world/mean", np.zeros(3))
    write_hdf5(stats, "/world/scale", np.ones(3))
    assert E.check_stats(stats, "world") is None
    assert "melspc" in E.check_stats(stats, "melspc")
    args = E.get_parser().parse_args(["--waveforms", "w", "--feats", "f", "--checkpoint", "a.pkl", "b.pkl",
                                      "--outfile", "o.tsv"])
    assert args.checkpoint == ["a.pkl", "b.pkl"] and args.batch_samples > 0 and args.start is None
    rc = subprocess.run([sys.executable, "-m", "pytorchwavenetvocoder_b200.bin.evaluate", "--waveforms", str(a),
                         "--feats", str(b), "--checkpoint", "c.pkl", "--outfile", str(tmp_path / "o.tsv")],
                        cwd=ROOT, capture_output=True, text=True)
    assert rc.returncode == 1 and "2 waveforms but 1" in rc.stderr
    assert not os.path.exists(tmp_path / "o.tsv")


def test_train_dev_flag_refusals():
    from pytorchwavenetvocoder_b200.bin.train import check_dev_args, get_parser
    base = ["--waveforms", "w", "--feats", "f", "--stats", "s", "--expdir", "e"]
    p = get_parser()
    assert check_dev_args(p.parse_args(base)) is None
    assert p.parse_args(base).dev_interval == 0
    assert "go together" in check_dev_args(p.parse_args(base + ["--dev_waveforms", "d"]))
    assert "go together" in check_dev_args(p.parse_args(base + ["--dev_feats", "d"]))
    assert "needs --dev_waveforms" in check_dev_args(p.parse_args(base + ["--dev_interval", "5"]))
    assert check_dev_args(p.parse_args(base + ["--dev_interval", "-1"])) is not None
    assert check_dev_args(p.parse_args(base + ["--dev_waveforms", "d", "--dev_feats", "g", "--dev_interval", "5"])) \
        is None


# ---- the ordered gather under gloo ------------------------------------------------------------------------------------
def _gather_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pytorchwavenetvocoder_b200.parallel import gather_scores, shard_utterances
    from pytorchwavenetvocoder_b200.utils.scoring import corpus_mean
    rng = np.random.RandomState(7)
    nll_all, cnt_all = rng.standard_normal(11) * 1e3, rng.randint(0, 9, size=11)
    mine = shard_utterances(list(range(11)), world, rank)
    nll, cnt = gather_scores(nll_all[mine], cnt_all[mine])
    q.put((rank, nll, cnt, corpus_mean(nll, cnt)))
    dist.destroy_process_group()


def test_gather_scores_in_list_order():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 28500 + (os.getpid() % 1000)
    world = 3
    ps = [ctx.Process(target=_gather_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = sorted([q.get(timeout=120) for _ in ps], key=lambda r: r[0])
    for p in ps:
        p.join(60)
        assert p.exitcode == 0
    rng = np.random.RandomState(7)
    nll_all, cnt_all = rng.standard_normal(11) * 1e3, rng.randint(0, 9, size=11)
    one = S.corpus_mean(nll_all, cnt_all)
    for _, nll, cnt, cm in res:
        assert np.array_equal(nll, nll_all) and np.array_equal(cnt, cnt_all)
        assert cm[0] == one[0] and cm[1] == one[1] and (cm[2] == one[2] or np.isnan(one[2]))


def test_gather_scores_without_group():
    from pytorchwavenetvocoder_b200.parallel import gather_scores
    n, c = gather_scores([1.0, 2.0], [3, 4])
    assert n.dtype == np.float64 and c.dtype == np.int64 and list(c) == [3, 4]


# ---- the kernel ------------------------------------------------------------------------------------------------------
def test_cross_entropy_rows_ptxas():
    src = os.path.join(ROOT, "pytorchwavenetvocoder_b200", "csrc", "score.cu")
    out = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                          "--fmad=true", "-Xptxas", "-v", "-c", src, "-o", os.devnull],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = [l for l in out.stderr.splitlines() if "cross_entropy_rows" in l or "registers" in l or "spill" in l]
    regs = [int(l.split("Used ")[1].split(" ")[0]) for l in out.stderr.splitlines() if "registers" in l]
    assert len(regs) == 2 and max(regs) <= 128, lines         # 512 threads per block need <= 128
    assert all(" 0 bytes spill stores, 0 bytes spill loads" in l for l in out.stderr.splitlines() if "spill" in l)


def test_cross_entropy_rows_refusals_without_gpu():
    from pytorchwavenetvocoder_b200 import _lib
    lib = _lib.load()
    n0 = _lib.launch_count()
    assert lib.wnb_cross_entropy_rows(None, None, None, 0, None, None, 1, 4, 256, None) != 0
    assert lib.wnb_cross_entropy_rows(1, 1, 1, -1, 1, None, 1, 4, 256, None) != 0
    assert lib.wnb_cross_entropy_rows(1, 1, 1, 0, 1, None, 0, 4, 256, None) != 0
    assert _lib.launch_count() == n0
