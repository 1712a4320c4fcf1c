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
