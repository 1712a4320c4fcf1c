# -*- coding: utf-8 -*-
"""Thread-block clusters in gemm_nt_tc (csrc/gemm_nt_tc.cu): the weight box multicast across CM = 1, 2, 4 CTAs must
not change a single bit of any output.

Each case runs one training step (forward, cross entropy, backward) of the same model on the same batch three times,
with WNB_NT_CLUSTER forcing CM = 1, 2 and 4 for every gemm_nt_tc launch, and compares logits, loss and every gradient
with torch.equal.  The paths reach all the launch kinds and epilogues of the kernel:
  - deferred-skip stack (tf32): skip GEMM (N = 256, two column blocks, ReLU), dZ_all (10 column blocks for 30 blocks
    of 64 channels), gate backward without z in modes 2 and 3, dx with two time-shifted segments and the split output
    (reduce-add of dhaux), time tiles walked in reverse;
  - per-block tf32 / bf16 (composed path, R = 256): the gate forward and backward with z over two half boxes, plain
    epilogues with bias / add / accumulate, the post network (bias, ReLU, mask, N from 32 to 256 so that both the one-
    and two-CTA-per-SM ring layouts run).
Batch shapes: T not a multiple of the 64-row tile, B = 1 and 3; time-tile counts that are not multiples of CM (a
partial last cluster group) and groups that straddle two batch rows (11 tiles per row).
"""
import os

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu

CASES = [
    # (Q, A, R, S, depth, repeat, ks, U), math, deferred skip, B, T
    ((256, 28, 64, 512, 10, 3, 2, 0), "tf32", True, 3, 700),     # 33 time tiles: 16 pairs + 1, 8 quads + 1
    ((256, 28, 64, 512, 10, 3, 2, 0), "tf32", True, 1, 333),     # 6 time tiles
    ((256, 28, 64, 256, 4, 2, 2, 0), "tf32", True, 3, 1000),     # L*R = 512: dZ_all in two 256-column blocks
    ((256, 28, 64, 96, 3, 1, 2, 0), "tf32", True, 1, 200),       # S = 96: N = 96 weight boxes, 24-row slices at CM = 4
    ((256, 28, 256, 256, 4, 1, 2, 0), "tf32", False, 3, 700),    # composed path: gate over two half boxes
    ((256, 28, 256, 256, 4, 1, 2, 0), "bf16", False, 1, 333),
    ((256, 28, 128, 128, 4, 2, 2, 0), "bf16", False, 3, 1000),
    ((256, 28, 64, 32, 2, 1, 2, 0), "tf32", False, 3, 130),      # S = 32: post network N = 32
]


def _step(cfg, params, math_mode, deferred, x, h, t):
    from pytorchwavenetvocoder_b200.nets import cross_entropy
    net = our_model(cfg, params, math_mode=math_mode).train()
    net.deferred_skip = deferred
    y = net(x, h)
    loss = cross_entropy(y, t, min(32, x.shape[1] // 4))
    loss.backward()
    torch.cuda.synchronize()
    return y.detach().clone(), loss.detach().clone(), {k: v.grad.clone() for k, v in net.named_parameters()
                                                       if v.grad is not None}


@pytest.mark.parametrize("c,math_mode,deferred,B,T", CASES)
def test_cluster_size_is_bit_identical(c, math_mode, deferred, B, T, monkeypatch):
    cfg = O.Config(*c)
    params = O.make_params(cfg, 5)
    rng = np.random.RandomState(7)
    x = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    t = torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda()
    h = torch.from_numpy(rng.standard_normal((B, cfg.n_aux, T)).astype(np.float32)).cuda()
    runs = {}
    for cm in ("1", "2", "4"):
        monkeypatch.setenv("WNB_NT_CLUSTER", cm)
        runs[cm] = _step(cfg, params, math_mode, deferred, x, h, t)
    y1, l1, g1 = runs["1"]
    assert torch.isfinite(l1).item()
    for cm in ("2", "4"):
        y, l, g = runs[cm]
        assert torch.equal(y, y1), cm
        assert torch.equal(l, l1), cm
        assert g.keys() == g1.keys()
        for k in g1:
            assert torch.equal(g[k], g1[k]), (cm, k)
