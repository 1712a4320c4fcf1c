# -*- coding: utf-8 -*-
"""CPU tier: pins the decode references of tests/decode_reference.py.

* teacher forcing: one whole-sequence forward reproduces the oracle's step-by-step fast generation (kernel size 2 and 3,
  with and without upsampling, seeds of 1 sample, shorter and longer than the receptive field, ragged lengths, and
  dilations that are not powers of two set on the config), and the float64 torch forward reproduces ``oracle.forward``;
* the same forward with ``dtype=torch.float32`` is a float32 evaluation: within float32 rounding of float64, not equal
  to it, and returned as float64;
* Philox4x32-10 against the Random123 known-answer vectors;
* the lane-scan sampler: under the old rule, uniforms placed in the gaps between lanes return an inadmissible class
  (Q-1); under the fixed rule no uniform does, over 10^4 logit vectors;
* ``oracle._pick`` never returns a class of zero probability.
"""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests import decode_reference as D


def _batch_order(outs, n_list, Q):
    """oracle.batch_fast_generate's completion-order outputs -> (B, max_n) in batch order, padded with Q // 2"""
    order = sorted(range(len(n_list)), key=lambda b: (n_list[b], b))
    gen = np.full((len(n_list), max(n_list)), Q // 2, np.int64)
    for o, b in zip(outs, order):
        gen[b, :n_list[b]] = o
    return gen


TF_CASES = [
    # (cfg tuple, T0, n_list, mode)
    ((256, 28, 16, 32, 3, 2, 3, 5), 4, [12, 7, 1], "argmax"),      # kernel 3, U = 5, 1 < T0 < rf
    ((256, 28, 16, 32, 3, 1, 2, 0), 30, [9, 9], "argmax"),          # T0 = 30 > rf = 8, aux at sample rate
    ((256, 28, 16, 32, 3, 2, 2, 4), 1, [10, 3, 6], "sampling"),     # T0 = 1, U = 4, ragged
    ((256, 31, 8, 24, 2, 2, 3, 0), 2, [1, 11], "sampling"),         # kernel 3, U = 0, A = 31
]


@pytest.mark.parametrize("case", range(len(TF_CASES)))
def test_teacher_forced_logits_match_fast_generate(case):
    t, T0, n_list, mode = TF_CASES[case]
    cfg = O.Config(*t)
    p = {k: v.astype(np.float64) for k, v in O.make_params(cfg, 40 + case).items()}
    rng = np.random.RandomState(case)
    B, n = len(n_list), max(n_list)
    U = max(cfg.upsampling_factor, 1)
    x = rng.randint(0, 256, size=(B, T0)).astype(np.int64)
    h = rng.standard_normal((B, cfg.n_aux, (n + T0 + U - 1) // U))
    uni = [rng.uniform(size=n).astype(np.float32) for _ in range(B)] if mode == "sampling" else None
    outs, lg = O.batch_fast_generate(cfg, p, x, h, n_list, mode=mode, uniforms=uni, return_logits=True)
    gen = _batch_order(outs, n_list, 256)
    for dev in (None, "cpu"):
        ref = D.teacher_forced_logits(cfg, p, x, h, gen, device=dev, chunk=2)
        assert ref.shape == lg.shape
        for b in range(B):
            err = np.abs(ref[b, :n_list[b]] - lg[b, :n_list[b]]).max()
            assert err <= 1e-12 * max(1.0, np.abs(lg).max()), (case, dev, b, err)


def test_teacher_forced_logits_follow_custom_dilations():
    """dilations replaced on the config (ks 4, 1 and one longer than the decode among them) reach both references"""
    cfg = O.Config(256, 28, 16, 32, 3, 2, 4, 0)
    cfg.dilations = [1, 3, 11, 2, 5, 6]
    cfg.receptive_field = 3 * sum(cfg.dilations) + 1
    p = {k: v.astype(np.float64) for k, v in O.make_params(cfg, 45).items()}
    rng = np.random.RandomState(4)
    n_list = [9, 4]
    x = rng.randint(0, 256, size=(2, 3)).astype(np.int64)
    h = rng.standard_normal((2, 28, 3 + 9))
    outs, lg = O.batch_fast_generate(cfg, p, x, h, n_list, mode="argmax", return_logits=True)
    gen = _batch_order(outs, n_list, 256)
    for dev in (None, "cpu"):
        ref = D.teacher_forced_logits(cfg, p, x, h, gen, device=dev)
        for b in range(2):
            assert np.abs(ref[b, :n_list[b]] - lg[b, :n_list[b]]).max() <= 1e-12 * max(1.0, np.abs(lg).max()), (dev, b)
    default = O.Config(*cfg.as_tuple())        # the power-of-two dilations give other logits
    assert np.abs(D.teacher_forced_logits(default, p, x, h, gen, device="cpu")[0, :9] - lg[0, :9]).max() > 1e-3


def test_forward64_float32_is_a_float32_evaluation():
    cfg = O.Config(256, 28, 16, 32, 4, 1, 3, 0)
    p = {k: v.astype(np.float64) for k, v in O.make_params(cfg, 3).items()}
    rng = np.random.RandomState(1)
    x = rng.randint(0, 256, size=(2, 50))
    h = rng.standard_normal((2, 28, 50))
    y64 = D.forward64(cfg, p, x, h)
    y32 = D.forward64(cfg, p, x, h, dtype=torch.float32)
    assert y32.dtype == np.float64 and y32.shape == y64.shape
    assert np.array_equal(y32, y32.astype(np.float32))          # every value is a float32
    err = np.abs(y32 - y64).max()
    assert 0 < err <= 64 * 2.0 ** -24 * max(1.0, np.abs(y64).max()), err
    sd = D.teacher_forced_logits(cfg, p, x[:, :5], h, x[:, 5:20], device="cpu", dtype=torch.float32)
    assert np.array_equal(sd, sd.astype(np.float32))
    with pytest.raises(AssertionError):
        D.teacher_forced_logits(cfg, p, x[:, :5], h, x[:, 5:20], dtype=torch.float32)


def test_forward64_matches_oracle_forward():
    cfg = O.Config(256, 28, 16, 32, 4, 1, 3, 0)
    p = {k: v.astype(np.float64) for k, v in O.make_params(cfg, 3).items()}
    rng = np.random.RandomState(1)
    x = rng.randint(0, 256, size=(2, 50))
    h = rng.standard_normal((2, 28, 50))
    assert np.abs(D.forward64(cfg, p, x, h) - O.forward(cfg, p, x, h)).max() < 1e-12


def test_philox_known_answers():
    """Random123 kat_vectors for philox4x32_10"""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = tuple(int(v) for v in D.philox4x32_10(ctr, key))
        assert got == want, ["%08x" % v for v in got]


def test_philox_uniform_layout():
    """counter (step, utt, 0, 0), key (seed lo, seed hi), 24-bit uniform; broadcasting agrees with scalar calls"""
    seed = 0x0123456789ABCDEF
    u = D.philox_uniform(seed, np.arange(5)[:, None], np.arange(7)[None, :])
    assert u.shape == (5, 7) and u.dtype == np.float32
    r = D.philox4x32_10((6, 4, 0, 0), (0x89ABCDEF, 0x01234567))
    assert u[4, 6] == np.float32((int(r[0]) >> 8) * 2.0 ** -24)
    assert u[2, 3] == D.philox_uniform(seed, 2, 3)
    assert np.all((u >= 0) & (u < 1)) and np.all(u * 2 ** 24 == np.round(u * 2 ** 24))


def _logit_rows(n, seed):
    rng = np.random.RandomState(seed)
    sig = rng.uniform(0.5, 4.0, size=(n, 1))
    return (rng.standard_normal((n, 256)) * sig).astype(np.float32)


def test_old_rule_gap_picks_and_fixed_rule_never():
    """10^4 logit vectors (normal, sigma 0.5-4): a uniform placed in a gap of the old rule's lane intervals returns
    class Q-1 outside the admissible set; the fixed rule returns an admissible class for the same uniform, for random
    uniforms and for 0 and 1 - 2^-24."""
    lg = _logit_rows(10000, 7)
    gaps = [(i, D.gap_uniform(lg[i])) for i in range(lg.shape[0])]
    gaps = [(i, u) for i, u in gaps if u is not None]
    assert len(gaps) >= 5000, len(gaps)            # most vectors have a gap the old rule leaves unclaimed
    idx = np.array([i for i, _ in gaps])
    ug = np.array([u for _, u in gaps], np.float32)
    ok = D.admissible(lg[idx], ug)
    old = D.emulate_pick(lg[idx], ug, "old")
    bad_old = ~ok[np.arange(idx.size), old]
    print("rows with a reachable gap: %d / %d; old rule inadmissible there: %d (all Q-1: %s)"
          % (idx.size, lg.shape[0], bad_old.sum(), bool(np.all(old[bad_old] == 255))))
    assert bad_old.mean() > 0.9 and np.all(old[bad_old] == 255)
    new = D.emulate_pick(lg[idx], ug, "fixed")
    assert ok[np.arange(idx.size), new].all()
    rng = np.random.RandomState(8)
    for u in (rng.randint(0, 2 ** 24, size=lg.shape[0]).astype(np.float32) * np.float32(2 ** -24),
              np.zeros(lg.shape[0], np.float32), np.full(lg.shape[0], 1 - 2 ** -24, np.float32)):
        new = D.emulate_pick(lg, u, "fixed")
        assert D.admissible(lg, u)[np.arange(lg.shape[0]), new].all()
        assert np.array_equal(new, D.emulate_pick(lg, u, "old"))   # no gap hit: the same picks as before the fix


def test_fixed_rule_at_every_lane_boundary():
    """the uniforms the GPU boundary sweep uses (+-8 ulps around each of the 31 lane boundaries): always admissible
    under the fixed rule, including rows whose tail classes have zero fp32 probability"""
    lg = _logit_rows(200, 9)
    lg[:50, 200:] = -200.0                        # e_q = 0 for the tail: never a legal pick
    lg[50:60, :8] = -200.0                        # a whole lane of zero probability
    n_old_bad = 0
    for r in range(lg.shape[0]):
        u = D.boundary_uniforms(lg[r])
        rows = np.repeat(lg[r:r + 1], u.size, 0)
        ok = D.admissible(rows, u)
        new = D.emulate_pick(rows, u, "fixed")
        assert ok[np.arange(u.size), new].all(), r
        n_old_bad += int((~ok[np.arange(u.size), D.emulate_pick(rows, u, "old")]).sum())
    assert n_old_bad > 0
    # a target at or past the total (uni = 1) picks the last class of nonzero probability
    row = lg[0:1]
    assert D.emulate_pick(row, np.ones(1, np.float32), "fixed")[0] == 199
    assert D.emulate_pick(row, np.ones(1, np.float32), "old")[0] == 255


def test_admissible_set():
    lg = np.zeros((1, 256), np.float32)
    lg[0, 10] = 20.0                              # e^20: class 10 holds all but 5e-7 of the mass
    lg[0, 255] = -200.0
    a = D.admissible(lg, np.array([0.5], np.float32))[0]
    assert list(np.nonzero(a)[0]) == [10]
    a = D.admissible(lg, np.array([1.0], np.float32))[0]
    assert not a[255] and a[254]


def test_oracle_pick_never_returns_zero_probability():
    row = np.zeros(256, np.float32)
    row[250:] = -200.0
    assert O._pick(row, "sampling", 1.0) == 249
    assert O._pick(row, "sampling", 1 - 2 ** -24) <= 249
    assert O._pick(row, "sampling", 0.0) == 0
    lg = _logit_rows(300, 10)
    rng = np.random.RandomState(11)
    for r in range(lg.shape[0]):
        u = np.float32(rng.uniform())
        k = O._pick(lg[r], "sampling", u)
        assert D.admissible(lg[r:r + 1], np.array([u]))[0, k]
