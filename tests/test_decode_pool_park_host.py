# -*- coding: utf-8 -*-
"""CPU tier: parking and cancelling streams of a decode pool (``DecodePool(park_below=m)``, ``cancel``) without a GPU.

* scripted ``PoolSchedule`` calls under ``park_below`` 1 and 3: a starved stream parked and resumed into another slot, a
  resumed stream served ahead of an older waiting stream, a partly starved stream parked under m = 3 and not under
  m = 1, cancelling a waiting, an active and a parked stream, and ``park_below=None`` giving today's calls;
* ``PoolSchedule`` with parking drives the float FIFO oracle as ``DecodePool`` drives the bf16 decoder: a parked row is
  copied into a compact store with the rotation ``v - g0`` (slot s of the row to slot (s + v - g0) mod qlen) and back
  into any free row with ``g0' - v``, its last ks codes kept aside.  Streams stall for several calls, resume into other
  rows, are cancelled, and a lowered ``POOL_COUNTER_LIMIT`` rebases g while streams are parked.  Every stream that is
  not cancelled must reproduce ``oracle.batch_fast_generate`` exactly, and a cancelled one a prefix of it;
* the three park entry points reject bad shapes, slots, dilations and pointers before touching a device;
* decode_bf16_park.cu compiles for sm_90a without spills and without a C7510 / C7513 note."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import wavenet_oracle as O
from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.nets import wavenet as W
from tests.test_decode_pool_host import _upsampled

DIL = [1, 2, 4, 1, 2, 4]   # rf 15 at ks 2; with U 4 a one-sample seed needs frame f for samples 4f .. 4f + 3


def _desc(call):
    return dict(g0=call.g0, n=call.n, rows=[(slot, st.sid, i0, c) for slot, st, i0, c in call.rows],
                admit=[(T0, [st.sid for st in grp]) for T0, grp in call.admit], finished=call.finished,
                park=[(slot, st.sid, r) for slot, st, r in call.park],
                resume=[(slot, st.sid, r) for slot, st, r in call.resume])


def test_park_then_resume_into_another_slot():
    s = W.PoolSchedule(2, 15, DIL, 2, 4, park_below=1)
    a, b, c = s.add(0, 1, 10), s.add(1, 1, 10), s.add(2, 1, 6)
    a.frames = b.frames = 1
    call = _desc(s.next_call())
    assert call["rows"] == [(0, 0, 0, 4), (1, 1, 0, 4)] and call["g0"] == 1 and not call["park"]
    c.frames, b.frames = 2, 2                               # a starves; c complete; b can run 4 more
    call = _desc(s.next_call())
    # a's next position is P - 1 + 4 = 18 at step g0 = 5: it parks with rotation 13, and c takes its row
    assert call["park"] == [(0, 0, 13)] and call["admit"] == [(1, [2])] and call["resume"] == []
    assert call["rows"] == [(0, 2, 0, 4), (1, 1, 4, 4)] and call["n"] == 4 and s.parked == [a] and a.slot is None
    a.frames = 3                                            # a complete; b starves
    call = _desc(s.next_call())
    assert call["park"] == [(1, 1, 22 - 9)] and call["resume"] == [(1, 0, 9 - 18)]     # a resumes into b's row
    assert call["rows"] == [(0, 2, 4, 2), (1, 0, 4, 6)] and call["finished"] == [2, 0] and s.parked == [b]
    b.frames = 3
    call = _desc(s.next_call())
    assert call["resume"] == [(0, 1, 15 - 22)] and call["rows"] == [(0, 1, 8, 2)] and call["finished"] == [1]
    assert s.next_call() is None and not s.streams and not s.parked and s.slots == [None, None]


def test_resumed_stream_goes_ahead_of_an_older_waiting_stream():
    s = W.PoolSchedule(2, 15, DIL, 2, 4, park_below=1)
    w, a, c = s.add(0, 1, 10), s.add(1, 1, 10), s.add(2, 1, 30)
    a.frames = c.frames = 1                                 # w, the oldest, has no frames yet
    call = _desc(s.next_call())
    assert call["admit"] == [(1, [1, 2])] and call["rows"] == [(0, 1, 0, 4), (1, 2, 0, 4)]
    assert s.next_call() is None and s.slots == [a, c] and not s.parked   # nobody runs: nothing is parked either
    c.frames = 8                                            # c complete; a starves
    call = _desc(s.next_call(max_samples=5))
    assert call["park"] == [(0, 1, 18 - 5)] and call["rows"] == [(1, 2, 4, 5)] and s.slots == [None, c]
    w.frames, a.frames = 1, 2                               # both could take the one free row: a was parked, it goes first
    call = _desc(s.next_call(max_samples=5))
    assert call["resume"] == [(0, 1, 10 - 18)] and call["admit"] == [] and s.waiting == [w]
    assert call["rows"] == [(0, 1, 4, 4), (1, 2, 9, 4)] and call["n"] == 4


@pytest.mark.parametrize("m", [1, 3])
def test_partly_starved_stream_parks_under_3_not_1(m):
    s = W.PoolSchedule(2, 15, DIL, 2, 4, park_below=m)
    a, b = s.add(0, 1, 20), s.add(1, 1, 20)
    a.frames, b.frames = 1, 3
    call = _desc(s.next_call(max_samples=2))
    assert call["rows"] == [(0, 0, 0, 2), (1, 1, 0, 2)]
    call = _desc(s.next_call())                             # a can run 2 samples, b 10
    if m == 1:
        assert call["park"] == [] and call["n"] == 2 and call["rows"] == [(0, 0, 2, 2), (1, 1, 2, 2)]
    else:
        assert call["park"] == [(0, 0, 16 - 3)] and call["n"] == 10 and call["rows"] == [(1, 1, 2, 10)]
        a.frames, b.frames = 2, 5                           # a: 6 runnable >= 3, resumed; b complete
        call = _desc(s.next_call())
        assert call["resume"] == [(0, 0, 13 - 16)] and call["rows"] == [(0, 0, 2, 6), (1, 1, 12, 6)]


def test_waiting_stream_needs_min_m_samples():
    s = W.PoolSchedule(1, 15, DIL, 2, 4, park_below=5)
    a, b = s.add(0, 1, 3), s.add(1, 1, 20)
    a.frames, b.frames = 1, 1                               # a needs min(5, 3) = 3 and can run 3; b can run 4 < 5
    call = _desc(s.next_call())
    assert call["admit"] == [(1, [0])] and call["rows"] == [(0, 0, 0, 3)] and call["finished"] == [0]
    assert s.next_call() is None and s.waiting == [b]
    b.frames = 2
    assert _desc(s.next_call())["rows"] == [(0, 1, 0, 8)]


def test_cancel_waiting_active_and_parked():
    s = W.PoolSchedule(2, 15, DIL, 2, 4, park_below=1)
    a, b, c, d = s.add(0, 1, 10), s.add(1, 1, 10), s.add(2, 1, 10), s.add(3, 1, 10)
    a.frames = b.frames = 1
    s.next_call()
    s.cancel(2)                                             # waiting
    assert s.waiting == [d] and 2 in s.finished and 2 not in s.streams
    b.frames = 2                                            # a starves: parked; d has no frames, so row 0 stays free
    call = _desc(s.next_call())
    assert call["park"] == [(0, 0, 13)] and call["rows"] == [(1, 1, 4, 4)] and s.slots == [None, b]
    s.cancel(0)                                             # parked
    assert s.parked == [] and a.slot is None
    s.cancel(1)                                             # active: its row is free for the next call
    assert s.slots == [None, None] and s.finished == {0, 1, 2}
    with pytest.raises(KeyError):
        s.cancel(1)
    d.frames = 1
    call = _desc(s.next_call())
    assert call["admit"] == [(1, [3])] and call["rows"] == [(0, 3, 0, 4)] and not call["park"] and not call["resume"]
    s.cancel(3)
    assert s.next_call() is None and not s.streams and s.finished == {0, 1, 2, 3}


def test_park_below_none_is_lock_step():
    """test_decode_pool_host.py::test_schedule_rules's script, with park_below=None given: the same calls, no parking"""
    s = W.PoolSchedule(2, 15, DIL, 2, 4, park_below=None)
    a, b, c = s.add(0, 1, 10), s.add(1, 1, 3), s.add(2, 1, 5)
    calls = []
    b.frames = 1
    calls.append(s.next_call())
    a.frames, c.frames = 1, 3
    calls.append(s.next_call(max_samples=2))
    calls.append(s.next_call())
    assert s.next_call() is None                            # a starves: no launch, c waits too
    a.frames = 3
    calls.append(s.next_call())
    got = [_desc(c) for c in calls]
    assert [(d["g0"], d["n"]) for d in got] == [(1, 3), (4, 2), (6, 2), (8, 6)]
    assert [d["rows"] for d in got] == [[(0, 1, 0, 3)], [(0, 0, 0, 2), (1, 2, 0, 2)], [(0, 0, 2, 2), (1, 2, 2, 2)],
                                        [(0, 0, 4, 6), (1, 2, 4, 1)]]
    assert all(d["park"] == [] and d["resume"] == [] for d in got)
    assert W.PoolSchedule(2, 15, DIL, 2, 4).park_below is None
    for bad in (0, -1, 1.5, "2"):
        with pytest.raises(ValueError):
            W.PoolSchedule(2, 15, DIL, 2, 4, park_below=bad)


def _park_run(cfg, p, streams, capacity, mode, seed, m, cancel_after):
    """Decode ``streams`` [(x (T0,), total, h (A, nf), uniforms (total,), arrival, stall)] through PoolSchedule with
    ``park_below=m`` and the oracle; stream k gets no frames during the iterations in ``stall`` and is cancelled once it
    has ``cancel_after[k]`` samples.  Returns ({stream: samples}, every g0, [(stream, call it parked in, call it resumed in,
    slot it left, slot it entered)])."""
    rng = np.random.RandomState(seed)
    Q, ks, U = cfg.n_quantize, cfg.kernel_size, cfg.upsampling_factor
    Uc = max(U, 1)
    dtype = p["causal.conv.weight"].dtype
    sched = W.PoolSchedule(capacity, cfg.receptive_field, cfg.dilations, ks, U, park_below=m)
    pool = O.FifoState(cfg, capacity, dtype)
    qmax = max(q.shape[2] for q in pool.q)
    shift = sched.period * (qmax // sched.period + 2)
    hist = [[Q // 2] * ks for _ in range(capacity)]
    got, sent, g0s = {}, {}, []
    stores = {}        # id -> (per-layer (R, qlen) store, last ks codes, parked at g0, from slot)
    moves = []
    it = 0
    while len(sched.finished) < len(streams):
        for k, (x, total, h, _, arrival, stall) in enumerate(streams):
            if arrival == it:
                sched.add(k, len(x), total)
                got[k], sent[k] = [], 0
            if k in cancel_after and k in sched.streams and len(got[k]) >= cancel_after[k]:
                sched.cancel(k)
                stores.pop(k, None)
            if k in sched.streams and sent[k] < h.shape[1] and it not in stall:
                F = min(int(rng.randint(0, 4 if U == 0 else 2)), h.shape[1] - sent[k])   # frames of U > 0 hold U samples
                sent[k] += F
                sched.streams[k].frames += F
        it += 1
        assert it < 5000
        call = sched.next_call(None if rng.rand() < 0.3 else int(rng.randint(1, 8)))
        if call is None:
            continue
        g0s.append(call.g0)
        for slot, st, rot in call.park:                     # the row into a store of the stream's own positions
            assert st.position - rot == call.g0
            store = [np.zeros_like(q[slot]) for q in pool.q]
            for q_pool, q_st in zip(pool.q, store):
                qlen = q_st.shape[1]
                for s in range(qlen):
                    q_st[:, (s + rot) % qlen] = q_pool[slot, :, s]
            stores[st.sid] = (store, hist[slot][-ks:], len(g0s) - 1, slot)
            for q_pool in pool.q:
                q_pool[slot] = np.nan                       # whoever takes the row next must rewrite every slot
        for T0, group in call.admit:
            P = max(T0, cfg.receptive_field)
            n_pad = P - T0
            scratch = O.FifoState(cfg, len(group), dtype)
            seq = [np.array([Q // 2 if pos < n_pad else streams[st.sid][0][pos - n_pad] for st in group])
                   for pos in range(P)]
            hup = [_upsampled(cfg, p, streams[st.sid][2]) for st in group]
            for pos in range(P - 1):
                col = max(pos - n_pad, 0)
                prev = [seq[pos - (ks - 1 - j)] if pos - (ks - 1 - j) >= 0 else -np.ones(len(group), np.int64)
                        for j in range(ks - 1)]
                O.fifo_step(cfg, p, scratch, prev, seq[pos], np.stack([hh[:, col] for hh in hup]).astype(dtype),
                            want_logits=False)
            for b, st in enumerate(group):
                for q_pool, q_new in zip(pool.q, scratch.q):
                    qlen = q_new.shape[2]
                    for s in range(qlen):
                        q_pool[st.slot, :, (s + call.g0 - (P - 1)) % qlen] = q_new[b, :, s]
                hist[st.slot] = [int(seq[P - ks + j][b]) for j in range(ks)]
        for slot, st, rot in call.resume:                   # the store into any free row
            assert call.g0 - rot == st.P - 1 + {r[1].sid: r[2] for r in call.rows}[st.sid]   # its first sample is step g0
            store, tail, g_park, from_slot = stores.pop(st.sid)
            for q_pool, q_st in zip(pool.q, store):
                qlen = q_st.shape[1]
                q_pool[slot] = np.nan                       # every slot must be rewritten
                for s in range(qlen):
                    q_pool[slot, :, (s + rot) % qlen] = q_st[:, s]
            hist[slot] = list(tail)
            moves.append((st.sid, g_park, len(g0s) - 1, from_slot, slot))
        rows = {slot: (st, i0, c) for slot, st, i0, c in call.rows}
        for k in range(call.n):
            hcol = np.zeros((capacity, cfg.n_aux), dtype)
            for slot, (st, i0, c) in rows.items():
                assert c == call.n or st.done == st.total, "an unfinished stream in a row ran fewer steps than the call"
                if k < c:
                    col = st.aux_column(i0 + k)
                    assert col < sent[st.sid] * Uc, "a call used an aux column that had not arrived"
                    hcol[slot] = _upsampled(cfg, p, streams[st.sid][2])[:, col]
            pool.pos = call.g0 + k + shift
            prev = [np.array([hist[s][-ks + j] for s in range(capacity)]) for j in range(ks - 1)]
            lg = O.fifo_step(cfg, p, pool, prev, np.array([hist[s][-1] for s in range(capacity)]), hcol)
            for s in range(capacity):
                pick = 0
                if s in rows and k < rows[s][2]:
                    st, i0, _ = rows[s]
                    pick = O._pick(lg[s], mode, streams[st.sid][3][i0 + k])
                    got[st.sid].append(pick)
                hist[s].append(pick)
    return got, g0s, moves


def _stalling_streams(cfg, n, seed):
    rng = np.random.RandomState(seed)
    rf, U = cfg.receptive_field, max(cfg.upsampling_factor, 1)
    out = []
    for k in range(n):
        T0 = [1, 5, rf + 3][k % 3]
        total = int(rng.randint(16, 48))
        nf = (T0 - 1 + total + U - 1) // U + 1
        x = rng.randint(0, cfg.n_quantize, size=T0).astype(np.int64)
        h = rng.standard_normal((cfg.n_aux, nf)).astype(np.float32)
        arrival = int(rng.randint(0, 12))
        stall = set()
        for _ in range(3):                                  # three stalls of 3 .. 10 iterations after arrival
            a = arrival + int(rng.randint(1, 16))
            stall |= set(range(a, a + int(rng.randint(3, 11))))
        out.append((x, total, h, rng.uniform(size=total).astype(np.float32), arrival, stall))
    return out


@pytest.mark.parametrize("ks", [2, 3])
@pytest.mark.parametrize("U", [0, 4])
@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("m", [1, 3])
def test_parking_schedule_reproduces_one_shot(ks, U, mode, m, monkeypatch):
    cfg = O.Config(32, 5, 8, 12, 3, 2, ks, U)
    p = O.make_params(cfg, 7 * ks + U)
    streams = _stalling_streams(cfg, 12, 3 * ks + U + m)
    period = W.PoolSchedule(3, cfg.receptive_field, cfg.dilations, ks, U).period
    monkeypatch.setattr(W, "POOL_COUNTER_LIMIT", ks - 1 + period + 23)
    cancel_after = {4: 1, 9: 0}                             # one mid-stream, one before it starts
    got, g0s, moves = _park_run(cfg, p, streams, 3, mode, 5 * ks + U + m, m, cancel_after)
    for k, (x, total, h, uni, _, _) in enumerate(streams):
        want = O.batch_fast_generate(cfg, p, x[None], h[None], [total], mode, [uni])[0].tolist()
        if k in cancel_after:
            assert got[k] == want[:len(got[k])] and cancel_after[k] <= len(got[k]) < total, k
        else:
            assert got[k] == want, k
    assert len(moves) >= 4, moves
    assert any(a != b for _, _, _, a, b in moves), moves                         # resumed into another row
    # g rebased while a stream was parked
    assert any(any(b < a for a, b in zip(g0s[cp:cr], g0s[cp + 1:cr + 1])) for _, cp, cr, _, _ in moves), (moves, g0s)


def _ptrs(n, base=16):
    return (ctypes.c_void_p * max(n, 1))(*[base * (k + 1) for k in range(n)])


def test_park_bytes():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 30)(*([2 ** k for k in range(10)] * 3))
    assert lib.wnb_decode_bf16_park_bytes(512, 2, dil, 30) == 3069 * 512 * 2       # arctic 512/256: 3.1 MB
    assert lib.wnb_decode_bf16_park_bytes(256, 3, dil, 30) == 2 * 3069 * 256 * 2
    assert lib.wnb_decode_bf16_park_bytes(512, 2, None, 30) == 0
    assert lib.wnb_decode_bf16_park_bytes(512, 1, dil, 30) == 0
    assert lib.wnb_decode_bf16_park_bytes(512, 2, (ctypes.c_int32 * 2)(1, 0), 2) == 0


@pytest.mark.parametrize("fn", ["wnb_decode_bf16_pool_park", "wnb_decode_bf16_pool_unpark"])
def test_park_entry_points_reject_bad_arguments_without_gpu(fn):
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)
    name = fn[len("wnb_"):].encode()

    def call(q=16, cap=8, slots=(7, 0), stores="ok", rot=(-5, 9), n=2, R=512, ks=2, dl=dil, L=2):
        arr = lambda v: None if v is None else (ctypes.c_int32 * max(len(v), 1))(*v)
        st = _ptrs(2) if stores == "ok" else stores
        if fn.endswith("_park"):
            return lib.wnb_decode_bf16_pool_park(q, cap, arr(slots), st, arr(rot), n, R, ks, dl, L, None)
        return lib.wnb_decode_bf16_pool_unpark(st, q, cap, arr(slots), arr(rot), n, R, ks, dl, L, None)

    def fails(what, **kw):
        assert call(**kw) == -1, kw
        err = lib.wnb_last_error()
        assert name in err and what in err, (kw, err)

    for kw in (dict(cap=0), dict(n=0), dict(n=65), dict(R=0), dict(R=96), dict(ks=1), dict(L=0), dict(L=65)):
        fails(b"bad shape", **kw)
    for kw in (dict(q=None), dict(slots=None), dict(stores=None), dict(rot=None), dict(dl=None),
               dict(stores=(ctypes.c_void_p * 2)(16, None))):
        fails(b"null pointer", **kw)
    fails(b"not 16-byte aligned", stores=(ctypes.c_void_p * 2)(16, 40))
    for kw in (dict(slots=(8, 0)), dict(slots=(0, -1))):
        fails(b"slot", **kw)
    fails(b"slot 3 given twice", slots=(3, 3))
    fails(b"dilations must be positive", dl=(ctypes.c_int32 * 2)(1, 0))


def test_park_kernels_compile_without_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    assert "decode_bf16_park.cu" in build.SOURCES
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "decode_bf16_park.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    assert not [line for line in text.splitlines() if "C7510" in line or "C7513" in line], text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, re.S):
        found[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert len(found) == 2 and all("park_kernel" in k for k in found), found
    assert all(v == (0, 0) for v in found.values()), found
