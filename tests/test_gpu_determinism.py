# -*- coding: utf-8 -*-
"""GPU tier: the same inputs give the same results, bit for bit, run after run -- a tf32 training step of the
deferred-skip stack and an fp32 (SIMT) training step of the per-block path (every gradient, including the reductions
over time that CTAs share), and a sampling-mode decode."""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu


def _training_step_gradients_identical_across_runs(cfg, math_mode):
    p = O.make_params(cfg, 8)
    rng = np.random.RandomState(3)
    B, T = 2, 4096
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, 28, T // 16)).astype(np.float32)).cuda()
    runs = []
    for _ in range(3):
        net = our_model(cfg, p, math_mode=math_mode).train()
        loss = net.forward_loss(x, h, t, 64)
        loss.backward()
        runs.append((loss.item(), {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None}))
    for loss, grads in runs[1:]:
        assert loss == runs[0][0]
        for k, g in runs[0][1].items():
            assert torch.equal(g, grads[k]), k


def test_training_step_gradients_identical_across_runs():
    _training_step_gradients_identical_across_runs(O.Config(256, 28, 64, 128, 6, 2, 2, 16), "tf32")


def test_fp32_training_step_gradients_identical_across_runs():
    """the SIMT weight and bias gradients are split over (batch, time range) CTAs whose partial sums are added in slot
    order, so they do not depend on which CTA finishes first"""
    _training_step_gradients_identical_across_runs(O.Config(256, 28, 128, 96, 4, 2, 3, 16), "fp32")


def test_sampling_decode_identical_across_runs():
    cfg = O.Config(256, 28, 64, 512, 10, 3, 2, 80)
    net = our_model(cfg, O.make_params(cfg, 5)).eval()
    rng = np.random.RandomState(6)
    # 64 utterances: the two-CTA cluster form of the warp kernel, as in the benchmark
    x = torch.full((64, 1), 128, dtype=torch.int64).cuda()
    h = torch.from_numpy(rng.standard_normal((64, 28, 251)).astype(np.float32)).cuda()
    with torch.no_grad():
        a = net._decode(x, h, [20000] * 64, "sampling", seed=1234).cpu()
        b = net._decode(x, h, [20000] * 64, "sampling", seed=1234).cpu()
    assert torch.equal(a, b)
