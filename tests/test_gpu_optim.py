# -*- coding: utf-8 -*-
"""GPU tier: pytorchwavenetvocoder_b200.optim.Adam (one wnb_adam_flat launch per step) against torch.optim.Adam -- the
reference's optimizer (bin/train.py:457-460) -- on identical gradients, through the real training step, and through a
checkpoint round trip in torch's own state_dict format."""
import copy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


class _Holder(torch.nn.Module):
    """parameters of mixed shapes whose gradients are slices of one flat buffer, as nets.WaveNet's backward leaves them"""

    def __init__(self, shapes, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(*s, generator=g)) for s in shapes])

    def set_grads(self, seed):
        g = torch.Generator().manual_seed(seed)
        n = sum(p.numel() for p in self.ps)
        flat = (torch.randn(n, generator=g) * torch.rand(n, generator=g) * 0.1).cuda()
        off = 0
        for p in self.ps:
            p.grad = flat[off:off + p.numel()].view(p.shape)
            off += p.numel()
        self._wnb_flat_grad = flat


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_matches_torch_adam_on_identical_gradients(wd):
    from pytorchwavenetvocoder_b200.optim import Adam
    shapes = [(64, 256, 2), (64,), (128, 64, 2), (3,), (512, 64, 1), (1, 1, 1, 80), (1,), (256, 512, 1)]   # (sizes not all % 4)
    a, b = _Holder(shapes, 0).cuda(), _Holder(shapes, 0).cuda()
    ours = Adam(a.parameters(), lr=1e-3, weight_decay=wd, module=a)
    ref = torch.optim.Adam(b.parameters(), lr=1e-3, weight_decay=wd)
    for it in range(12):
        a.set_grads(100 + it)
        b.set_grads(100 + it)
        ours.step()
        ref.step()
    assert ours.flat_steps == 12
    for p, q in zip(a.ps, b.ps):
        err = (p - q).abs().max().item()
        assert err <= 2e-6 * max(q.abs().max().item(), 1.0), err
        so, sr = ours.state[p], ref.state[q]
        for key in ("exp_avg", "exp_avg_sq"):    # (a few ulp of the largest entry: lerp vs the two-step form, fma contraction)
            assert (so[key] - sr[key]).abs().max().item() <= 2e-6 * sr[key].abs().max().item(), key
        assert float(so["step"]) == 12.0
    # parameters without a gradient are left alone (torch.optim.Adam skips them; the last block's res_1x1 is such a one)
    c = _Holder(shapes, 1).cuda()
    frozen = torch.nn.Parameter(torch.ones(5, device="cuda"))
    o3 = Adam(list(c.parameters()) + [frozen], lr=1e-2, module=c)
    c.set_grads(7)
    o3.step()
    assert o3.flat_steps == 1 and torch.equal(frozen, torch.ones(5, device="cuda"))


def test_checkpoint_round_trip_in_torch_format_and_fallback():
    from pytorchwavenetvocoder_b200.optim import Adam
    shapes = [(32, 16), (7,), (64, 8, 2)]
    a = _Holder(shapes, 3).cuda()
    ours = Adam(a.parameters(), lr=2e-3, module=a)
    for it in range(3):
        a.set_grads(it)
        ours.step()
    sd = copy.deepcopy(ours.state_dict())
    assert set(sd["state"][0].keys()) == {"step", "exp_avg", "exp_avg_sq"}
    # (1) torch's Adam loads our state and continues exactly as we do
    b = _Holder(shapes, 3).cuda()
    b.load_state_dict(a.state_dict())
    ref = torch.optim.Adam(b.parameters(), lr=2e-3)
    ref.load_state_dict(copy.deepcopy(sd))
    # (2) a fresh optimizer of ours resumes from the same checkpoint
    c = _Holder(shapes, 3).cuda()
    c.load_state_dict(a.state_dict())
    res = Adam(c.parameters(), lr=2e-3, module=c)
    res.load_state_dict(copy.deepcopy(sd))
    for it in range(3, 6):
        for m in (a, b, c):
            m.set_grads(it)
        ours.step(); ref.step(); res.step()
    for p, q, r in zip(a.ps, b.ps, c.ps):
        assert (p - q).abs().max().item() <= 2e-6 and torch.equal(p, r)
    assert res.flat_steps == 3 and float(res.state[c.ps[0]]["step"]) == 6.0
    # gradients that are NOT slices of one buffer: torch's own step runs (and the step counters stay right)
    for p in a.ps:
        p.grad = torch.randn_like(p)
    a._wnb_flat_grad = None
    before = ours.flat_steps
    ours.step()
    assert ours.flat_steps == before and all(float(ours.state[p]["step"]) == 7.0 for p in a.ps)


def test_training_step_through_the_real_model():
    """nets.WaveNet (stack path) + optim.Adam: the flat path is taken, the loss falls, the state_dict keeps the reference's
    keys and shapes, and the result equals torch.optim.Adam's to rounding."""
    from oracle import wavenet_oracle as O
    from tests.util import our_model
    from pytorchwavenetvocoder_b200.optim import Adam
    cfg = O.Config(256, 28, 64, 64, 3, 2, 2, 4)
    p = O.make_params(cfg, 5)
    rng = np.random.RandomState(0)
    x = torch.from_numpy(rng.randint(0, 256, size=(2, 512)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(2, 512)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((2, 28, 128)).astype(np.float32)).cuda()
    nets, opts, losses = [], [], [[], []]
    for which in range(2):
        net = our_model(cfg, p)
        net.math_mode = "tf32"
        net.train()
        nets.append(net)
        opts.append(Adam(net.parameters(), lr=1e-3, module=net) if which == 0 else torch.optim.Adam(net.parameters(), lr=1e-3))
    shapes = {k: tuple(v.shape) for k, v in nets[0].state_dict().items()}
    for it in range(8):
        for which in range(2):
            loss = nets[which].forward_loss(x, h, t, cfg.receptive_field)
            opts[which].zero_grad(set_to_none=True)
            loss.backward()
            opts[which].step()
            losses[which].append(loss.item())
    assert opts[0].flat_steps == 8
    assert losses[0][-1] < losses[0][0] - 0.05
    assert {k: tuple(v.shape) for k, v in nets[0].state_dict().items()} == shapes
    assert max(abs(a - b) for a, b in zip(losses[0], losses[1])) < 2e-3      # (tf32 gradients are not run-to-run identical)


# ------------------------------------------------------------------------------------------------------------------
# wnb_adam_flat element by element against float64 (tests/adam_reference.py): the torch comparisons above test
# compatibility, these test accuracy
# ------------------------------------------------------------------------------------------------------------------
from tests import adam_reference as A                      # noqa: E402
from tests.test_gpu_tc_stages import _report                # noqa: E402

STEPS = (1, 2, 10, 100000)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid_stride_floats():
    """floats one pass of adam_flat_kernel's float4 loop covers: 4 per thread, 256 threads, 8 blocks per SM"""
    return 4 * 256 * 8 * _sms()


def _adam_call(p, g, m, v, n, lr, betas, eps, wd, bc1, bc2):
    from pytorchwavenetvocoder_b200 import _lib
    P = _lib.ptr
    _lib.check(_lib.load().wnb_adam_flat(P(p) if torch.is_tensor(p) else p, P(g), P(m), P(v), n, lr, betas[0], betas[1],
                                         eps, wd, bc1, bc2, _lib.stream()), "adam_flat")


def _check_step(before, g, after, sc, where, res):
    """after = one step from before (dicts p/m/v of numpy fp32) within the float64 chain; exact where nothing moves"""
    ref, bound = A.adam_step(before["p"], g, before["m"], before["v"], sc)
    for key, (r, i) in A.ratios(after, ref, bound).items():
        res[key] = max(res.get(key, 0.0), r)
        assert r <= 1.0, "%s: %s[%d] err/bound %.3g (got %r, float64 %r, bound %.3g; p %r g %r m %r v %r)" % (
            where, key, i, r, float(after[key][i]), ref[key][i], bound[key][i], float(before["p"][i]), float(g[i]),
            float(before["m"][i]), float(before["v"][i]))
    still = (g == 0) & (before["m"] == 0) & (before["v"] == 0) & ((sc["wd"] == 0) | (before["p"] == 0))
    assert np.array_equal(after["p"][still].view(np.int32), before["p"][still].view(np.int32)), where
    assert np.all(after["m"][still] == 0) and np.all(after["v"][still] == 0), where


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("betas,eps", [((0.9, 0.999), 1e-8), ((0.9, 0.999), 1e-3), ((0.5, 0.9), 1e-8),
                                       ((0.5, 0.9), 1e-3)])
@pytest.mark.parametrize("size", ["1", "3", "4", "7", "3_passes"])
def test_adam_flat_elementwise_against_float64(size, betas, eps, wd):
    """one step per bias correction (steps 1, 2, 10, 10^5) on values spread over 23 decades, first steps (m = v = 0),
    all-zero entries and p = 0; n = 1, 3, 7 run the tail loop alone, 4 the float4 loop alone, and 2 * (4 * 256 * 8 *
    SMs) + 5 runs the grid-stride loop three times and the tail"""
    n = 2 * _grid_stride_floats() + 5 if size == "3_passes" else int(size)
    res = {}
    for k in STEPS:
        bc1, bc2 = A.bias_corrections(betas, k)
        sc = A.scalars(1e-3, betas, eps, wd, bc1, bc2)
        p, g, m, v = A.spread_inputs(n, 17 * k + n)
        if n <= 7:                     # the few elements of the small sizes: a first step, a zero entry, p = 0
            p, g, m, v = (np.resize(a, n) for a in A.spread_inputs(8 * n, k))
            m[0] = v[0] = 0.0
            if n > 2:
                g[2] = m[2] = v[2] = 0.0
        dev = [torch.from_numpy(a.copy()).cuda() for a in (p, g, m, v)]
        _adam_call(*dev, n, 1e-3, betas, eps, wd, bc1, bc2)
        after = dict(p=dev[0].cpu().numpy(), m=dev[2].cpu().numpy(), v=dev[3].cpu().numpy())
        assert torch.equal(dev[1].cpu(), torch.from_numpy(g))
        _check_step(dict(p=p, m=m, v=v), g, after, sc, "n %d step %d" % (n, k), res)
    _report("adam n=%d betas=%s eps=%g wd=%g" % (n, betas, eps, wd), res)


def test_adam_flat_rejects_bad_arguments():
    from pytorchwavenetvocoder_b200 import _lib
    buf = [torch.ones(64, device="cuda") for _ in range(4)]
    p0 = buf[0].clone()
    with pytest.raises(_lib.WnbError, match="empty"):
        _adam_call(*buf, 0, 1e-3, (0.9, 0.999), 1e-8, 0.0, 0.1, 0.001)
    with pytest.raises(_lib.WnbError, match="aligned"):
        _adam_call(buf[0].data_ptr() + 4, *buf[1:], 60, 1e-3, (0.9, 0.999), 1e-8, 0.0, 0.1, 0.001)
    for bc1, bc2 in ((0.0, 0.001), (0.1, 0.0), (-0.1, 0.001), (0.1, -1e-3)):
        with pytest.raises(_lib.WnbError, match="bias corrections"):
            _adam_call(*buf, 64, 1e-3, (0.9, 0.999), 1e-8, 0.0, bc1, bc2)
    torch.cuda.synchronize()
    assert torch.equal(buf[0], p0) and torch.equal(buf[2], p0) and torch.equal(buf[3], p0)


def _set_flat_grad(holder, flat):
    off = 0
    for q in holder.ps:
        q.grad = flat[off:off + q.numel()].view(q.shape)
        off += q.numel()
    holder._wnb_flat_grad = flat


def _step_checked(opt, holder, grad, where, res):
    """one optim.Adam step on `grad`, checked against the float64 chain from a snapshot of the flat p / m / v taken just
    before it, with the bias corrections of the step count the optimizer is about to use"""
    f = opt._flat
    if f is None:                                            # first step: laid out (or resumed) inside step()
        before = None
    else:
        before = {k: f[k].cpu().numpy().copy() for k in ("p", "m", "v")}
        k_next = f["k"] + 1
    _set_flat_grad(holder, grad)
    if before is None:
        st = [opt.state.get(q, {}) for q in holder.ps]
        before = dict(p=torch.cat([q.detach().reshape(-1) for q in holder.ps]).cpu().numpy(),
                      m=np.concatenate([s["exp_avg"].reshape(-1).cpu().numpy() if "exp_avg" in s else
                                        np.zeros(q.numel(), np.float32) for s, q in zip(st, holder.ps)]),
                      v=np.concatenate([s["exp_avg_sq"].reshape(-1).cpu().numpy() if "exp_avg_sq" in s else
                                        np.zeros(q.numel(), np.float32) for s, q in zip(st, holder.ps)]))
        k_next = max([int(float(s["step"])) for s in st if "step" in s] + [0]) + 1
    flat_before = opt.flat_steps
    opt.step()
    assert opt.flat_steps == flat_before + 1
    f, grp = opt._flat, opt.param_groups[0]
    assert f["k"] == k_next and float(f["step_t"]) == float(k_next)
    betas = grp["betas"]
    sc = A.scalars(grp["lr"], betas, grp["eps"], grp["weight_decay"], *A.bias_corrections(betas, k_next))
    after = {k: f[k].cpu().numpy() for k in ("p", "m", "v")}
    _check_step(before, grad.cpu().numpy(), after, sc, "%s step %d" % (where, k_next), res)


@pytest.mark.parametrize("rem", [1, 2, 3])
def test_optim_adam_steps_against_float64_and_resume_at_step_1e5(rem):
    """optim.Adam on a flat buffer of (grid-stride threshold + 4j + rem) floats: several steps, each against the float64
    chain; then a fresh optimizer resumes from a state_dict at step 10^5 (k = max(k, step)) and is checked the same way"""
    from pytorchwavenetvocoder_b200.optim import Adam
    n = _grid_stride_floats() + 4 * 1001 + rem
    shapes = [(37,), (n // 128 - 1, 64, 2), (n - 37 - (n // 128 - 1) * 128,)]
    assert sum(int(np.prod(s)) for s in shapes) == n and n % 4 == rem
    a = _Holder(shapes, rem).cuda()
    opt = Adam(a.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, module=a)
    res = {}
    for it in range(4):
        g = torch.from_numpy(A.spread_inputs(n, 100 * rem + it)[1]).cuda()
        _step_checked(opt, a, g, "n %d" % n, res)
    sd = copy.deepcopy(opt.state_dict())
    rng = np.random.RandomState(rem)
    for i, st in sd["state"].items():
        st["step"] = torch.tensor(1e5)
        st["exp_avg"] = torch.from_numpy(A.spread_inputs(st["exp_avg"].numel(), i)[2]).view_as(st["exp_avg"]).cuda()
        st["exp_avg_sq"] = torch.from_numpy(
            (10.0 ** rng.uniform(-30, 4, st["exp_avg_sq"].numel())).astype(np.float32)).view_as(st["exp_avg_sq"]).cuda()
    b = _Holder(shapes, rem + 10).cuda()
    res_opt = Adam(b.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, module=b)
    res_opt.load_state_dict(sd)
    for it in range(3):
        g = torch.from_numpy(A.spread_inputs(n, 7 + it)[1]).cuda()
        _step_checked(res_opt, b, g, "resumed n %d" % n, res)
    assert res_opt._flat["k"] == 100003
    _report("optim.Adam n=%d" % n, res)
