# -*- coding: utf-8 -*-
"""CPU tier: the static work split of the weight-gradient kernel (wnb_wgrad_partition, a pure host function).

Each problem is cut into its fixed time chunks (the summation order of its gradient) and every chunk is placed whole on
exactly one CTA; CTAs end one problem and start the next, zero-stage problems and CTAs without work are handled,
locked problems (operands shared through L2) run as equal time chunks side by side, the split is the same on every
call, and no CTA's cost exceeds the larger of the mean and its locked chunk by more than one chunk."""
import ctypes

import numpy as np
import pytest


def _lib():
    from pytorchwavenetvocoder_b200 import _lib as L_
    return L_.load()


def partition(stages, nchunk, cost, lock, sms, max_pieces=4096):
    lib = _lib()
    n = len(stages)
    st = (ctypes.c_int * max(n, 1))(*stages)
    nc = (ctypes.c_int * max(n, 1))(*nchunk)
    co = (ctypes.c_double * max(n, 1))(*cost)
    lk = (ctypes.c_int * max(n, 1))(*lock)
    first = (ctypes.c_int * (sms + 1))()
    pcs = (ctypes.c_int * (3 * max_pieces))()
    np_ = lib.wnb_wgrad_partition(st, nc, co, lk, n, sms, first, pcs, max_pieces)
    assert np_ >= 0, lib.wnb_last_error()
    pieces = [tuple(pcs[3 * i:3 * i + 3]) for i in range(np_)]
    return list(first), pieces


def chunks(n, k):
    """the chunks of an n-stage problem cut k ways: ceil(n / k) stages each, empty ones dropped"""
    per = -(-n // k)
    return [(min(n, j * per), min(n, (j + 1) * per)) for j in range(k) if min(n, j * per) < min(n, (j + 1) * per)]


def stack_like(L, ntiles, sms=132, skip_sets=40):
    """the stack's list at the bench shape: dW1 (L segments), dW2res (L-1), dWskip (locked M-block x column group
    sets), chunked as the kernel's host code does (SMs / problems of the call) with its per-stage costs (us)"""
    stages = [ntiles] * (L + (L - 1) + skip_sets)
    nchunk = [max(1, sms // L)] * L + [max(1, sms // (L - 1))] * (L - 1) + [max(1, sms // skip_sets)] * skip_sets
    cost = [1.03] * L + [0.60] * (L - 1) + [1.21] * skip_sets
    lock = [0] * (2 * L - 1) + [1] * skip_sets
    return stages, nchunk, cost, lock


def check_cover(stages, nchunk, first, pieces, sms):
    """every problem's chunks appear exactly once, whole, and nothing else"""
    assert first[0] == 0 and first[sms] == len(pieces)
    assert all(first[j] <= first[j + 1] for j in range(sms))
    got = sorted(pieces)
    want = sorted((i, s0, s1) for i, (n, k) in enumerate(zip(stages, nchunk)) for s0, s1 in chunks(n, k))
    assert got == want


def cta_costs(cost, first, pieces, sms):
    return [sum((s1 - s0) * cost[p] for p, s0, s1 in pieces[first[j]:first[j + 1]]) for j in range(sms)]


@pytest.mark.parametrize("sms", [132, 114])
def test_stack_list_covers_balances_and_locks(sms):
    L, ntiles = 30, 8 * 721
    stages, nchunk, cost, lock = stack_like(L, ntiles, sms)
    first, pieces = partition(stages, nchunk, cost, lock, sms)
    check_cover(stages, nchunk, first, pieces, sms)
    tot = cta_costs(cost, first, pieces, sms)
    mean = sum(s * c for s, c in zip(stages, cost)) / sms
    biggest = max((s1 - s0) * cost[p] for p, s0, s1 in pieces if not lock[p])
    locked_load = [sum((s1 - s0) * cost[p] for p, s0, s1 in pieces[first[j]:first[j + 1]] if lock[p]) for j in range(sms)]
    assert max(tot) <= max(mean, max(locked_load)) + biggest + 1e-9, (max(tot), mean)
    # the locked sets: chunk c of set i on CTA c * 40 + i, every CTA of a chunk on the same time range; CTAs of odd
    # chunks run their other chunks first
    nl = 40
    k = sms // nl
    for j in range(nl * k):
        mine = pieces[first[j]:first[j + 1]]
        lp = [x for x in mine if lock[x[0]]]
        assert len(lp) == 1
        i, c = 2 * L - 1 + j % nl, j // nl
        assert lp[0] == (i,) + chunks(ntiles, k)[c]
        assert (mine.index(lp[0]) == 0) == (c % 2 == 0 or len(mine) == 1)
    for j in range(nl * k, sms):
        assert not any(lock[p] for p, _, _ in pieces[first[j]:first[j + 1]])
    # CTAs end one problem and start the next
    assert any(len({p for p, _, _ in pieces[first[j]:first[j + 1]]}) > 1 for j in range(sms))


def test_same_on_every_call():
    stages, nchunk, cost, lock = stack_like(30, 5768)
    a = partition(stages, nchunk, cost, lock, 132)
    for _ in range(3):
        assert partition(stages, nchunk, cost, lock, 132) == a


@pytest.mark.parametrize("n,ntiles,k,sms", [(1, 1000, 132, 132), (7, 3, 3, 132), (64, 5, 2, 132), (3, 100, 5, 16)])
def test_unlocked_chunks(n, ntiles, k, sms):
    rng = np.random.RandomState(n + ntiles)
    stages, nchunk = [ntiles] * n, [k] * n
    cost = list(rng.uniform(0.5, 2.0, n))
    first, pieces = partition(stages, nchunk, cost, [0] * n, sms)
    check_cover(stages, nchunk, first, pieces, sms)
    tot = cta_costs(cost, first, pieces, sms)
    mean = sum(s * c for s, c in zip(stages, cost)) / sms
    assert max(tot) <= mean + max((s1 - s0) * cost[p] for p, s0, s1 in pieces) + 1e-9
    if len(pieces) < sms:   # fewer chunks than CTAs: the others get no work at all
        assert sum(first[j] == first[j + 1] for j in range(sms)) == sms - len(pieces)


def test_zero_stage_problems_empty_chunks_and_empty_ctas():
    stages = [0, 5, 0, 3, 0, 10]
    nchunk = [2, 4, 3, 1, 1, 4]          # 5 stages in 4 chunks of 2: one chunk empty; 10 in 4 of 3: 3+3+3+1
    cost = [1.0, 1.0, 2.0, 1.5, 1.0, 1.0]
    lock = [0, 0, 1, 0, 1, 0]
    first, pieces = partition(stages, nchunk, cost, lock, 16)
    check_cover(stages, nchunk, first, pieces, 16)
    assert not any(p in (0, 2, 4) for p, _, _ in pieces)
    assert sum(first[j] == first[j + 1] for j in range(16)) == 16 - len(pieces)
    first, pieces = partition([0, 0], [1, 1], [1.0, 1.0], [0, 1], 8)
    assert pieces == [] and first == [0] * 9
    first, pieces = partition([], [], [], [], 4)
    assert pieces == [] and first == [0] * 5


def test_locked_only_matches_equal_chunks():
    """one call with several M-blocks / column groups (the post network, the composed path): SMs // sets chunks per
    set, chunk c of set i on CTA c * sets + i, no other work"""
    stages, lock = [100] * 16, [1] * 16
    k = 132 // 16
    first, pieces = partition(stages, [k] * 16, [1.0] * 16, lock, 132)
    check_cover(stages, [k] * 16, first, pieces, 132)
    assert [pieces[first[j]] for j in range(16 * k)] == [(j % 16,) + chunks(100, k)[j // 16] for j in range(16 * k)]
    assert all(first[j] == first[j + 1] for j in range(16 * k, 132))
    # more locked chunks than CTAs: they are placed like the others, whole
    first, pieces = partition([10] * 20, [1] * 20, [1.0] * 20, [1] * 20, 8)
    check_cover([10] * 20, [1] * 20, first, pieces, 8)
    assert sorted(first[j + 1] - first[j] for j in range(8)) == [2, 2, 2, 2, 3, 3, 3, 3]


def test_rejects_bad_input_and_overflow():
    lib = _lib()
    first = (ctypes.c_int * 5)()
    st = (ctypes.c_int * 1)(-1)
    nc = (ctypes.c_int * 1)(4)
    co = (ctypes.c_double * 1)(1.0)
    lk = (ctypes.c_int * 1)(0)
    assert lib.wnb_wgrad_partition(st, nc, co, lk, 1, 4, first, None, 0) == -1
    st[0] = 100
    nc[0] = 0
    assert lib.wnb_wgrad_partition(st, nc, co, lk, 1, 4, first, None, 0) == -1
    nc[0] = 4
    pcs = (ctypes.c_int * 3)()
    assert lib.wnb_wgrad_partition(st, nc, co, lk, 1, 4, first, pcs, 1) == -1    # needs 4 pieces
    assert lib.wnb_wgrad_partition(st, nc, co, lk, 1, 4, first, None, 0) == 4     # counting only
