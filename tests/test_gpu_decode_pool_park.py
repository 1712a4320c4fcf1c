# -*- coding: utf-8 -*-
"""GPU tier: parking and cancelling streams of a bf16 decode pool (``WaveNet.decode_pool(park_below=m)``) keeps every
stream bit-identical to one-shot decoding.

80 or 160 streams per pool are fed aux frames slowly and withheld for stretches of calls, so streams park several times,
resume into other rows (other clusters at capacity 130) and at least one resumes after the pool has run more steps than
its longest queue holds.  Stream k must equal row k of ``net._decode(X, H, n_list, mode, seed=S, kernel="bf16")``
(``torch.equal``) in argmax and in Philox sampling, on arctic 512/256, the ljspeech-size shape (ks 3), 256/256 with 8
layers and the speaker-code shape (U 0).  Also: a park -> unpark round trip reproduces a row's slots bit for bit,
cancelled streams free their rows while the others stay exact, a counter rebase with parked streams, and the library
launches of a parking and a resuming call."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_decode_pool import ARCTIC, CASES, SHALLOW_256, _model, _one_shot, _streams

pytestmark = pytest.mark.gpu

# (capacity, streams, drive seed): at 130 rows, enough streams at once to fill rows of every cluster.  The schedule
# depends only on the host arithmetic, so the drive seeds are fixed ones whose schedules meet the coverage checks of
# test_parking_pool_equals_one_shot (at 130 rows a resume into another cluster is the rare one).
POOL = {"arctic": (64, 80, 64), "ljspeech_ks3": (64, 80, 79), "r256_L8": (130, 160, 167), "speaker_A31_U0": (64, 80, 85)}


def _trace(monkeypatch):
    """Record every PoolCall the pools make."""
    from pytorchwavenetvocoder_b200.nets import wavenet
    calls = []
    real = wavenet.PoolSchedule.next_call

    def traced(self, max_samples=None):
        call = real(self, max_samples)
        if call is not None:
            calls.append(call)
        return call
    monkeypatch.setattr(wavenet.PoolSchedule, "next_call", traced)
    return calls


def _stalls(streams, seed):
    """per stream: three stretches of 2 .. 40 calls after its arrival in which it gets no frames"""
    rng = np.random.RandomState(seed)
    out = []
    for _, _, _, arrival in streams:
        s = set()
        for _ in range(3):
            a = arrival + int(rng.randint(1, 40))
            s |= set(range(a, a + int(rng.randint(2, 41))))
        out.append(s)
    return out


def _run_parking_pool(net, streams, capacity, mode, seed, rng_seed, park_below, cancel_after=None):
    """Drive a parking pool; stream k is cancelled once it has cancel_after[k] samples.  Returns (pool, {k: codes})."""
    rng = np.random.RandomState(rng_seed)
    cancel_after = cancel_after or {}
    stalls = _stalls(streams, rng_seed + 1)
    Uc = max(net.upsampling_factor, 1)
    fmax = max(1, 100 // Uc) + 1                             # frames per call: up to about 100 samples
    pool = net.decode_pool(capacity, mode, seed, park_below=park_below)
    got = {k: [] for k in range(len(streams))}
    sent = [0] * len(streams)
    it = 0
    while it <= max(a for _, _, _, a in streams) or not all(pool.finished(k) for k in range(len(streams))):
        for k, (x, total, h, arrival) in enumerate(streams):
            if arrival == it:
                F = int(rng.randint(0, fmax))
                assert pool.admit(x, total, h[:, :F] if F else None, stream=k) == k
                sent[k] = F
            elif arrival < it and not pool.finished(k):
                if k in cancel_after and sum(c.numel() for c in got[k]) >= cancel_after[k]:
                    pool.cancel(k)
                    continue
                if sent[k] < h.size(1) and it not in stalls[k]:
                    F = min(int(rng.randint(0, fmax)), h.size(1) - sent[k])
                    pool.feed(k, h[:, sent[k]:sent[k] + F])
                    sent[k] += F
        it += 1
        assert it < 20000
        for k, codes in pool.step(None if rng.rand() < 0.2 else int(rng.randint(1, 150))).items():
            got[k].append(codes.cpu())
    return pool, {k: torch.cat(v) if v else torch.empty(0, dtype=torch.int32) for k, v in got.items()}


def _moves(calls):
    """[(stream, g0 of its park call, g0 of its resume call, slot left, slot entered)]"""
    parked, out = {}, []
    for call in calls:
        for slot, st, _ in call.park:
            parked[st.sid] = (call.g0, slot)
        for slot, st, _ in call.resume:
            g, s = parked.pop(st.sid)
            out.append((st.sid, g, call.g0, s, slot))
    return out


@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("case", list(CASES))
def test_parking_pool_equals_one_shot(case, mode, monkeypatch):
    cfg, net = _model(CASES[case])
    ci = list(CASES).index(case)
    capacity, nstreams, drive = POOL[case]
    streams = _streams(cfg, nstreams, 10 * ci + capacity + 3)
    seed = 2000 + ci
    want = _one_shot(net, streams, mode, seed)
    calls = _trace(monkeypatch)
    park_below = 1 if mode == "argmax" else 8
    pool, got = _run_parking_pool(net, streams, capacity, mode, seed, drive, park_below)
    assert not pool.active and not pool.waiting and not pool.parked
    for k in range(len(streams)):
        assert torch.equal(got[k], want[k]), (case, mode, k, int((got[k] != want[k]).sum()))
    moves = _moves(calls)
    qmax = (cfg.kernel_size - 1) * max(cfg.dilations)
    per_stream = {}
    for sid, *_ in moves:
        per_stream[sid] = per_stream.get(sid, 0) + 1
    assert len(moves) >= 10 and max(per_stream.values()) >= 2, moves            # streams park several times
    assert any(a != b for _, _, _, a, b in moves), moves                          # and resume into other rows
    assert max(gr - gp for _, gp, gr, _, _ in moves) >= qmax, (qmax, moves)       # after every queue has wrapped
    if capacity == 130:
        bc = -(-capacity // 3)
        assert any(a // bc != b // bc for _, _, _, a, b in moves), moves         # into another cluster


def _logical_rows(queues, capacity, R, nslots):
    """The pool workspace as [row][slot][channel] bf16 bit patterns (int16), the 128B swizzle undone."""
    ncl = -(-capacity // 64)
    bc = -(-capacity // ncl)
    q = queues.view(torch.int16).view(ncl, nslots, R // 64, 64, 8, 8)        # cluster, slot, tile, row, 16B chunk, bf16
    row = torch.arange(64, device=queues.device)
    phys = (torch.arange(8, device=queues.device)[None, :] ^ (row[:, None] & 7))   # chunk k of row r sits at k ^ (r & 7)
    q = torch.gather(q, 4, phys[None, None, None, :, :, None].expand(ncl, nslots, R // 64, 64, 8, 8))
    q = q.permute(0, 3, 1, 2, 4, 5).reshape(ncl, 64, nslots, R)[:, :bc]
    return q.reshape(ncl * bc, nslots, R)[:capacity]


def test_park_unpark_round_trip_is_bit_exact():
    from pytorchwavenetvocoder_b200 import _lib
    from pytorchwavenetvocoder_b200.nets.wavenet import ptr, stream
    lib = _lib.load()
    cfg, _ = _model(ARCTIC)
    R, ks, L, capacity = cfg.n_resch, cfg.kernel_size, len(cfg.dilations), 130
    dil = (ctypes.c_int32 * L)(*cfg.dilations)
    qlens = [(ks - 1) * d for d in cfg.dilations]
    nslots = sum(qlens)
    nbytes = lib.wnb_decode_bf16_park_bytes(R, ks, dil, L)
    assert nbytes == nslots * R * 2
    g = torch.Generator(device="cuda").manual_seed(5)
    queues = torch.randint(-128, 128, (lib.wnb_decode_bf16_workspace(capacity, R, ks, dil, L),), dtype=torch.int8,
                           device="cuda", generator=g).view(torch.uint8)
    before = _logical_rows(queues, capacity, R, nslots).clone()
    rng = np.random.RandomState(3)
    for n in (1, 7, 64):
        src = [int(v) for v in rng.choice(capacity, n, replace=False)]
        dst = [int(v) for v in rng.choice(capacity, n, replace=False)]
        rot = [int(v) for v in rng.randint(-100000, 100000, n)]
        stores = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(n)]
        arr = lambda v: (ctypes.c_int32 * n)(*v)
        _lib.check(lib.wnb_decode_bf16_pool_park(ptr(queues), capacity, arr(src),
                                                 (ctypes.c_void_p * n)(*[ptr(t) for t in stores]), arr(rot), n, R, ks,
                                                 dil, L, stream()), "park")
        # the store: layer l's row slot s at store slot (s + rot) mod qlen, plain [slot][R]
        for i in (0, n - 1):
            st = stores[i].view(torch.int16).view(nslots, R)
            q0 = 0
            for qlen in qlens:
                perm = [(s + rot[i]) % qlen for s in range(qlen)]
                assert torch.equal(st[q0 + torch.tensor(perm, device="cuda")], before[src[i], q0:q0 + qlen]), (n, i)
                q0 += qlen
        _lib.check(lib.wnb_decode_bf16_pool_unpark((ctypes.c_void_p * n)(*[ptr(t) for t in stores]), ptr(queues),
                                                   capacity, arr(dst), arr([-r for r in rot]), n, R, ks, dil, L,
                                                   stream()), "unpark")
        after = _logical_rows(queues, capacity, R, nslots)
        for i in range(n):
            assert torch.equal(after[dst[i]], before[src[i]]), (n, i)
        untouched = [r for r in range(capacity) if r not in dst]
        assert torch.equal(after[untouched], before[untouched]), n
        before = after.clone()


def test_cancel_frees_rows_and_keeps_others_exact():
    cfg, net = _model(SHALLOW_256)
    streams = _streams(cfg, 40, 91)
    want = _one_shot(net, streams, "sampling", 12)
    cancel_after = {k: streams[k][1] * f // 4 for k, f in ((3, 0), (10, 1), (17, 2), (25, 3))}
    pool, got = _run_parking_pool(net, streams, 8, "sampling", 12, 4, 1, cancel_after)
    assert not pool.active and not pool.waiting and not pool.parked
    cut = 0
    for k in range(len(streams)):
        if k in cancel_after:   # cut short, unless it finished in the call that passed cancel_after[k]
            assert torch.equal(got[k], want[k][:got[k].numel()]), k
            cut += got[k].numel() < want[k].numel()
        else:
            assert torch.equal(got[k], want[k]), k
    assert cut >= 2, cut
    for k in cancel_after:
        assert pool.finished(k)
        with pytest.raises(ValueError):
            pool.admit(streams[k][0], 10, stream=k)
        if got[k].numel() < want[k].numel():
            with pytest.raises(KeyError):
                pool.feed(k, torch.zeros(cfg.n_aux, 1, device="cuda"))
            with pytest.raises(KeyError):
                pool.cancel(k)


def test_cancel_active_waiting_and_parked_rows():
    cfg, net = _model(SHALLOW_256)
    g = torch.Generator(device="cuda").manual_seed(8)
    streams = [(torch.randint(0, 256, (1,), device="cuda", generator=g), 100,
                torch.randn(cfg.n_aux, 26, device="cuda", generator=g), 0) for _ in range(4)]
    want = _one_shot(net, streams, "argmax", 6)
    pool = net.decode_pool(2, "argmax", 6, park_below=1)
    got = {k: [] for k in range(4)}
    for k, (x, total, h, _) in enumerate(streams):
        pool.admit(x, total, h[:, :4], stream=k)                  # a one-sample seed: aux of samples 0 .. 15
    for k, c in pool.step().items():
        got[k].append(c.cpu())
    assert pool.active == [0, 1] and pool.waiting == [2, 3]
    pool.feed(1, streams[1][2][:, 4:])                          # 0 starves: parked, 2 takes its row
    for k, c in pool.step().items():
        got[k].append(c.cpu())
    assert pool.parked == [0] and pool.active == [2, 1] and pool.waiting == [3]
    pool.cancel(0)                                              # parked
    pool.cancel(1)                                              # active: its row is free for the next call
    pool.cancel(3)                                              # waiting
    assert pool.active == [2] and not pool.parked and not pool.waiting
    assert all(pool.finished(k) for k in (0, 1, 3))
    pool.feed(2, streams[2][2][:, 4:])
    while not pool.finished(2):
        for k, c in pool.step().items():
            got[k].append(c.cpu())
    assert [len(got[k]) for k in (0, 1, 3)] == [1, 2, 0]
    for k in range(4):
        g = torch.cat(got[k]) if got[k] else torch.empty(0, dtype=torch.int32)
        assert torch.equal(g, want[k][:g.numel()]), k
    assert torch.equal(torch.cat(got[2]), want[2])


def test_counter_rebase_with_parked_streams(monkeypatch):
    from pytorchwavenetvocoder_b200.nets import wavenet
    cfg, net = _model(SHALLOW_256)
    streams = _streams(cfg, 40, 78)
    want = _one_shot(net, streams, "sampling", 10)
    monkeypatch.setattr(wavenet, "POOL_COUNTER_LIMIT", 1 + 8 + 257)   # period 8: lcm of the queue lengths 1, 2, 4, 8
    calls = _trace(monkeypatch)
    _, got = _run_parking_pool(net, streams, 8, "sampling", 10, 6, 1)
    for k in range(len(streams)):
        assert torch.equal(got[k], want[k]), k
    g0s = [c.g0 for c in calls]
    parked, rebased_while_parked = set(), 0
    for a, b in zip(calls, calls[1:]):
        parked |= {st.sid for _, st, _ in a.park}
        parked -= {st.sid for _, st, _ in a.resume}
        if b.g0 < a.g0 and parked - {st.sid for _, st, _ in b.resume}:
            rebased_while_parked += 1
    assert rebased_while_parked >= 2, g0s


def test_launch_counts_of_parking_and_resuming_calls():
    """a parking call: the park launch, the inputs kernel and the decode; a resuming call: the unpark launch, the inputs
    kernel and the decode"""
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = _model(SHALLOW_256)
    pool = net.decode_pool(8, "sampling", 3, park_below=1)
    x = torch.zeros(1, dtype=torch.int64, device="cuda")
    h = torch.randn(28, 60, device="cuda")
    pool.admit(x, 200, h[:, :10])
    pool.admit(x, 200, h[:, :10])

    def counted(max_samples=None):
        l0 = _lib.launch_count()
        out = pool.step(max_samples)
        return _lib.launch_count() - l0, sorted(out)

    assert counted() == (18, [0, 1])                            # both admitted, 40 samples each
    pool.feed(1, h[:, 10:30])                                   # stream 0 starves
    assert counted(40) == (3, [1]) and pool.parked == [0]
    pool.feed(0, h[:, 10:20])
    assert counted() == (3, [0, 1]) and not pool.parked
    torch.cuda.synchronize()


def test_more_than_64_streams_park_and_resume_at_once():
    """100 streams of a 130-row pool park in one call and resume in one call: two launches of at most 64 rows each"""
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net = _model(SHALLOW_256)
    g = torch.Generator(device="cuda").manual_seed(11)
    streams = [(torch.randint(0, 256, (1,), device="cuda", generator=g), 120,
                torch.randn(cfg.n_aux, 31, device="cuda", generator=g), 0) for _ in range(101)]
    want = _one_shot(net, streams, "sampling", 21)
    pool = net.decode_pool(130, "sampling", 21, park_below=1)
    got = {k: [] for k in range(101)}

    def step():
        l0 = _lib.launch_count()
        for k, c in pool.step().items():
            got[k].append(c.cpu())
        return _lib.launch_count() - l0

    for k, (x, total, h, _) in enumerate(streams):
        pool.admit(x, total, h[:, :10], stream=k)                 # 40 samples of aux each
    step()
    pool.feed(100, streams[100][2][:, 10:20])                   # the other 100 starve
    assert step() == 4 and len(pool.parked) == 100 and pool.active == [100]
    for k in range(101):
        pool.feed(k, streams[k][2][:, 10 if k < 100 else 20:])
    assert step() == 4 and not pool.parked and not pool.active   # every stream complete: all finish in this call
    for k in range(101):
        assert torch.equal(torch.cat(got[k]), want[k]), k
