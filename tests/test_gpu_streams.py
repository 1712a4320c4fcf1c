# -*- coding: utf-8 -*-
"""GPU tier: the C ABI is safe for DISTINCT streams (SURVEY.md 8b): the block kernels' dynamic tile scheduler words are
owned by (device, stream), so two model forwards issued concurrently on two streams from two host threads give the
same logits as the same forwards run one after the other."""
import threading

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests.util import our_model

pytestmark = pytest.mark.gpu


def test_two_streams_two_threads_concurrent_forward():
    cfg = O.Config(256, 28, 64, 512, 6, 2, 2, 16)
    nets = [our_model(cfg, O.make_params(cfg, 30 + i), math_mode="tf32").eval() for i in range(2)]
    rng = np.random.RandomState(0)
    B, T = 4, 8192           # more tiles per launch than SMs: the dynamic scheduler is exercised
    xs = [torch.from_numpy(rng.randint(0, 256, size=(B, T)).astype(np.int64)).cuda() for _ in range(2)]
    hs = [torch.from_numpy(rng.standard_normal((B, 28, T // 16)).astype(np.float32)).cuda() for _ in range(2)]
    with torch.no_grad():
        want = [nets[i](xs[i], hs[i]).clone() for i in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    got = [None, None]
    errs = []

    def work(i):
        try:
            with torch.no_grad(), torch.cuda.stream(streams[i]):
                for _ in range(4):
                    got[i] = nets[i](xs[i], hs[i])
            streams[i].synchronize()
        except Exception as e:   # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t_ in th:
        t_.start()
    for t_ in th:
        t_.join()
    assert not errs, errs
    torch.cuda.synchronize()
    for i in range(2):
        assert torch.equal(got[i], want[i]), i     # same kernels, same tiles: bit-identical
