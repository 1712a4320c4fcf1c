# -*- coding: utf-8 -*-
"""CPU tier: the host side of resumable MLSA filtering (wnb_mlsa_filter_state, utils/mlsa.py MlsaStreamFilter) -- the
state size against the documented layout, argument checks made before any device work, and the key/slot bookkeeping
of MlsaStreamFilter (empty chunks launch nothing, so no GPU is needed)."""
import ctypes

import numpy as np
import pytest
import torch


def _lib():
    from pytorchwavenetvocoder_b200 import _lib
    return _lib, _lib.load()


@pytest.mark.parametrize("order", [2, 24, 59, 255])
@pytest.mark.parametrize("pd", [4, 5])
def test_state_size_matches_layout(order, pd):
    _, lib = _lib()
    # d1[1..pd], pt1[0..pd], pt20, pt[1..pd], then pd all-pass chains e[1..order]
    assert lib.wnb_mlsa_state_doubles(order, pd) == pd + (pd + 1) + 1 + pd + pd * order


@pytest.mark.parametrize("order,pd", [(1, 4), (256, 4), (24, 3), (24, 6)])
def test_state_size_rejects_what_the_filter_rejects(order, pd):
    _, lib = _lib()
    assert lib.wnb_mlsa_state_doubles(order, pd) == 0


def test_filter_state_rejects_bad_arguments():
    L, lib = _lib()
    fake = ctypes.c_void_p(256)            # never dereferenced: every case fails before any device work
    slots = (ctypes.c_int32 * 3)(0, 1, 2)

    def call(n_segs=3, order=24, alpha=0.41, pd=4, states=fake, n_slots=4, sl=slots, zero=None, x=fake):
        return lib.wnb_mlsa_filter_state(x, 1, fake, n_segs, fake, order, alpha, pd, 1.0, fake, 1, states, n_slots, sl,
                                         zero, None)

    def rejected(msg, **kw):
        assert call(**kw) != 0
        assert msg in lib.wnb_last_error(), lib.wnb_last_error()

    rejected(b"need a state table", states=None)                       # slot indices without a state table
    rejected(b"need a state table", sl=None)
    rejected(b"null pointer", x=None)
    rejected(b"slot 4 of 4", sl=(ctypes.c_int32 * 3)(0, 4, 1))          # slot out of range
    rejected(b"slot -1 of 4", sl=(ctypes.c_int32 * 3)(0, -1, 1))
    rejected(b"slot 1 given twice", sl=(ctypes.c_int32 * 3)(1, 0, 1))   # two segments racing on one slot
    rejected(b"need n_slots > 0", n_slots=0)
    rejected(b"pd must be 4 or 5", pd=3)
    rejected(b"pd must be 4 or 5", pd=6)
    rejected(b"2 <= order <= 255", order=1)
    rejected(b"2 <= order <= 255", order=256)
    rejected(b"2 <= order <= 255", n_segs=0)
    big = (ctypes.c_int32 * 1025)(*range(1025))
    rejected(b"n_segs <= 1024", n_segs=1025, sl=big, n_slots=2000)
    rejected(b"|alpha| must be < 1", alpha=1.0)


def _coef(order=24):
    from pytorchwavenetvocoder_b200.utils.mlsa import convert_mcep_to_mlsa_coef
    return convert_mcep_to_mlsa_coef(np.random.RandomState(0).randn(order + 1) * 0.6, 0.5, 0.41)


def test_stream_filter_bookkeeping():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.utils.mlsa import MlsaStreamFilter
    f = MlsaStreamFilter(_coef(), 0.41, 4, device="cpu")
    assert f.state_doubles == 3 * 4 + 2 + 4 * 24
    e16 = torch.zeros(0, dtype=torch.int16)
    out = f.filter({"a": e16, 7: e16, ("row", 2): e16})                 # empty chunks: keys open, no launch
    assert set(out) == {"a", 7, ("row", 2)} and all(v.numel() == 0 and v.dtype == torch.int16 for v in out.values())
    assert [f.slot(k) for k in ("a", 7, ("row", 2))] == [0, 1, 2]
    assert f.slot("b") is None
    f.close(7)
    assert f.slot(7) is None
    with pytest.raises(KeyError):
        f.close(7)
    f.filter({"b": e16, "c": e16})                                      # the freed slot goes to the first new key
    assert f.slot("b") == 1 and f.slot("c") == 3 and f.slot("a") == 0
    assert f.filter({}) == {}
    for k in range(70):                                                 # past the first table size
        f.filter({("n", k): torch.zeros(0, dtype=torch.float64)})
    assert sorted(f.slot(("n", k)) for k in range(70)) == list(range(4, 74))
    with pytest.raises(ValueError):
        f.filter({"a": torch.zeros(0, dtype=torch.float32)})
    with pytest.raises(ValueError):
        f.filter({"a": e16, "b": torch.zeros(0, dtype=torch.float64)})
    with pytest.raises(ValueError):
        f.filter({"a": torch.zeros(2, 3, dtype=torch.int16)})
    with pytest.raises(_lib.WnbError):                                  # samples on the CPU: no fallback
        f.filter({"a": torch.zeros(5, dtype=torch.int16)})
    with pytest.raises(ValueError):
        MlsaStreamFilter(_coef(), 0.41, 3, device="cpu")
    with pytest.raises(ValueError):
        MlsaStreamFilter(_coef(1), 0.41, 4, device="cpu")
