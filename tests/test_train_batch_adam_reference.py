# -*- coding: utf-8 -*-
"""CPU tier: the references the GPU tests hold wnb_make_train_batch (tests/loader_reference.py) and wnb_adam_flat
(tests/adam_reference.py) to run on CPU arrays, and they reject planted mistakes -- a comparison that a wrong kernel
could pass would prove nothing."""
import numpy as np
import pytest

from tests import adam_reference as A
from tests import loader_reference as L


def _scaler_data(seed=0, n=4096, D=28):
    rng = np.random.RandomState(seed)
    v = rng.standard_normal((n, D)) * 10.0 ** rng.uniform(-3, 3, (n, D))
    return v, rng.standard_normal(D) * 3, 0.1 + rng.rand(D) * 5


def test_scaler_modes_differ_and_mode_of_installed_sklearn():
    from sklearn.preprocessing import StandardScaler
    from pytorchwavenetvocoder_b200.utils.device_loader import _f32_scaler_mode
    v, mean, scale = _scaler_data()
    v32 = v.astype(np.float32)
    m0, m2 = L.apply_scaler(v32, mean, scale, "mode0"), L.apply_scaler(v32, mean, scale, "mode2")
    assert m0.dtype == m2.dtype == np.float32
    # the two float32 modes differ on this data, so a kernel that runs the other mode fails the GPU test
    assert np.count_nonzero(m0 != m2) > 100
    # a planted mistake: mode 0 computed in float32 arithmetic is mode 2, not mode 0
    wrong = (v32 - mean.astype(np.float32)) / scale.astype(np.float32)
    assert not np.array_equal(wrong, m0)
    # mode 0 without the intermediate rounding to float32 is also caught
    assert not np.array_equal(((v32.astype(np.float64) - mean) / scale).astype(np.float32), m0)
    # the installed scikit-learn is one of the two, and the probe names the right one
    sc = StandardScaler()
    sc.mean_, sc.scale_ = mean, scale
    mode = _f32_scaler_mode()
    assert np.array_equal(sc.transform(v32), {0: m0, 2: m2}[mode])
    assert np.array_equal(sc.transform(v).astype(np.float32), L.apply_scaler(v, mean, scale, "f64"))


@pytest.mark.parametrize("name", sorted(L.RING_CASES))
def test_ring_cases_reach_their_edges_and_a_clamped_index_is_caught(name):
    c = L.ring_case(name)
    rng = np.random.RandomState(1)
    fos = L.fos_ring(c) if c["fos"] else None
    assert set(c["reaches"]) <= L.windows_reach(c, fos), name
    codes = rng.randint(0, 256, c["cap_s"]).astype(np.int64)
    feat = rng.standard_normal((c["cap_f"], c["D"])).astype(np.float32)
    x, t, h = L.make_train_batch(codes, feat, fos, c["s0"], c["hop"], c["U"], c["cap_s"], c["cap_f"], None, None,
                                 c["B"], c["T"], c["Tf"], "f32_none")
    assert np.array_equal(x[:, 1:], t[:, :-1])
    # a plain per-element loop of the same formulas
    for b in range(c["B"]):
        so = c["s0"] + b * c["hop"]
        for i in (0, c["T"] // 2, c["T"] - 1):
            assert x[b, i] == codes[(so + i) % c["cap_s"]] and t[b, i] == codes[(so + i + 1) % c["cap_s"]]
        for j in (0, c["Tf"] - 1):
            row = (int(fos[(so + j) % c["cap_s"]]) if c["fos"] else so // c["U"] + j) % c["cap_f"]
            assert np.array_equal(h[b, :, j], feat[row])
    # a planted mistake: the sample index clamped instead of wrapped (in bounds, right for windows inside the ring)
    i = np.arange(c["T"] + 1)
    bad = np.stack([codes[np.minimum((c["s0"] + b * c["hop"]) % c["cap_s"] + i, c["cap_s"] - 1)] for b in range(c["B"])])
    assert not np.array_equal(bad[:, :-1], x) or not np.array_equal(bad[:, 1:], t)


@pytest.mark.parametrize("mu", [256, 1024])
def test_mulaw_restatement_matches_the_oracle_away_from_edges(mu):
    from oracle.wavenet_oracle import encode_mu_law
    from tests.golden.cases import mulaw_edge_mask, mulaw_pcm16_domain
    x = np.concatenate([mulaw_pcm16_domain(), L.mulaw_near_edges(mu), np.float32([1, -1, 0, -0.0])])
    got, want = L.mulaw_f32_reference(x, mu), encode_mu_law(x, mu)
    mask = L.mulaw_edge_mask_mu(x, mu)
    if mu == 256:
        assert np.array_equal(mask, mulaw_edge_mask(x))
    assert got.min() == 0 and got.max() == mu - 1
    assert not np.any((got != want) & ~mask), np.nonzero((got != want) & ~mask)
    assert np.abs(got - want).max() <= 1


def test_adam_bound_holds_for_fp32_arithmetic_and_rejects_planted_mistakes():
    worst = 0.0
    for betas in [(0.9, 0.999), (0.5, 0.9)]:
        for eps in [1e-8, 1e-3]:
            for wd in [0.0, 0.01]:
                for k in [1, 2, 10, 100000]:
                    sc = A.scalars(1e-3, betas, eps, wd, *A.bias_corrections(betas, k))
                    p, g, m, v = A.spread_inputs(20011, k)
                    ref, bound = A.adam_step(p, g, m, v, sc)
                    for contract in (False, True):
                        r = A.ratios(A.emulate_fp32(p, g, m, v, sc, contract=contract), ref, bound)
                        worst = max(worst, max(x for x, _ in r.values()))
                    # eps added before the bias correction: caught at step 1 (small |g|, eps not negligible)
                    bad = A.ratios(A.emulate_fp32(p, g, m, v, sc, eps_first=True), ref, bound)
                    if k == 1 and betas[1] == 0.999:
                        assert bad["p"][0] > 1, (betas, eps, wd)
                    # an update skipped (the tail loop not run) is caught
                    assert A.ratios(dict(p=p, m=m, v=v), ref, bound)["p"][0] > 1
                    # 1 - b2 rounded in float32 arithmetic instead of once from double
                    sc2 = dict(sc, omb2=float(np.float32(1) - np.float32(betas[1])))
                    if betas[1] == 0.999:
                        assert A.ratios(A.emulate_fp32(p, g, m, v, sc2), ref, bound)["v"][0] > 1
    assert worst <= 1.0, worst
