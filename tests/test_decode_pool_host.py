# -*- coding: utf-8 -*-
"""CPU tier: the continuous-batching decode pool (``DecodePool``) without a GPU.

* ``nets.wavenet.PoolSchedule`` (the host arithmetic every ``DecodePool.step`` uses) drives the float FIFO oracle
  (``oracle.FifoState`` / ``fifo_step``) as the pool drives the bf16 decoder: one FIFO batch of ``capacity`` rows stepped
  at the pool's global counter g, each admitted stream's warm-up run on its own and its queues moved into its row with the
  slot rotation ``(s + g0 - (P - 1)) mod (ks - 1) d``, each row given its own stream's aux column and uniform.  Streams
  arrive at different calls, have ragged lengths, seeds of one sample, shorter than and longer than the receptive field,
  aux in random chunks and ``max_samples`` windows; more streams than rows, so rows are reused; and a lowered
  ``POOL_COUNTER_LIMIT`` makes g rebase mid-stream.  Every stream must reproduce ``oracle.batch_fast_generate`` exactly,
  and every aux column a call uses must have arrived before it;
* the two pool entry points reject bad shapes, rows, slots, dilations and pointers before touching a device;
* decode_bf16_pool.cu compiles for sm_90a without spills and without a C7510 / C7513 note."""
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


def _upsampled(cfg, p, h):
    if cfg.upsampling_factor > 0:
        return O.upsample(h[None], p["upsampling.conv.weight"], p["upsampling.conv.bias"])[0]
    return h


def _pool_run(cfg, p, streams, capacity, mode, seed):
    """Decode ``streams`` [(x (T0,), total, h (A, nf), uniforms (total,), arrival)] through PoolSchedule and the oracle.
    Returns ({stream: samples}, every g0, the slots each stream took)."""
    rng = np.random.RandomState(seed)
    Q, ks, U = cfg.n_quantize, cfg.kernel_size, cfg.upsampling_factor
    Uc = max(U, 1)
    dtype = p["causal.conv.weight"].dtype
    sched = W.PoolSchedule(capacity, cfg.receptive_field, cfg.dilations, ks, U)
    pool = O.FifoState(cfg, capacity, dtype)
    qmax = max(q.shape[2] for q in pool.q)
    shift = sched.period * (qmax // sched.period + 2)   # same slots as g, and no tap before 0 for fifo_step's guard
    hist = [[Q // 2] * ks for _ in range(capacity)]
    got, sent, g0s, slots = {}, {}, [], {}
    it = 0
    while len(sched.finished) < len(streams):
        for k, (x, total, h, _, arrival) in enumerate(streams):
            if arrival == it:
                sched.add(k, len(x), total)
                got[k], sent[k] = [], 0
            if k in sched.streams and sent[k] < h.shape[1]:
                F = min(int(rng.randint(0, 4)), h.shape[1] - sent[k])
                sent[k] += F
                sched.streams[k].frames += F
        it += 1
        call = sched.next_call(None if rng.rand() < 0.3 else int(rng.randint(1, 8)))
        if call is None:
            continue
        g0s.append(call.g0)
        for T0, group in call.admit:
            P = max(T0, cfg.receptive_field)
            n_pad = P - T0
            scratch = O.FifoState(cfg, len(group), dtype)
            seq = [np.array([Q // 2 if pos < n_pad else streams[st.sid][0][pos - n_pad] for st in group])
                   for pos in range(P)]
            hup = [_upsampled(cfg, p, streams[st.sid][2]) for st in group]
            for pos in range(P - 1):
                col = max(pos - n_pad, 0)
                assert all(col < sent[st.sid] * Uc for st in group)
                prev = [seq[pos - (ks - 1 - j)] if pos - (ks - 1 - j) >= 0 else -np.ones(len(group), np.int64)
                        for j in range(ks - 1)]
                O.fifo_step(cfg, p, scratch, prev, seq[pos], np.stack([hh[:, col] for hh in hup]).astype(dtype),
                            want_logits=False)
            for b, st in enumerate(group):
                slots.setdefault(st.sid, []).append(st.slot)
                for q_pool, q_new in zip(pool.q, scratch.q):
                    qlen = q_new.shape[2]
                    for s in range(qlen):
                        q_pool[st.slot, :, (s + call.g0 - (P - 1)) % qlen] = q_new[b, :, s]
                hist[st.slot] = [int(seq[P - ks + j][b]) for j in range(ks)]
        rows = {slot: (st, i0, c) for slot, st, i0, c in call.rows}
        for k in range(call.n):
            hcol = np.zeros((capacity, cfg.n_aux), dtype)
            for slot, (st, i0, c) in rows.items():
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
    return got, g0s, slots


def _streams(cfg, n, seed):
    rng = np.random.RandomState(seed)
    rf, U = cfg.receptive_field, max(cfg.upsampling_factor, 1)
    out = []
    for k in range(n):
        T0 = [1, 5, rf + 3][k % 3]
        total = int(rng.randint(1, 26))
        nf = (T0 - 1 + total + U - 1) // U + 1
        x = rng.randint(0, cfg.n_quantize, size=T0).astype(np.int64)
        h = rng.standard_normal((cfg.n_aux, nf)).astype(np.float32)
        out.append((x, total, h, rng.uniform(size=total).astype(np.float32), int(rng.randint(0, 12))))
    return out


@pytest.mark.parametrize("ks", [2, 3])
@pytest.mark.parametrize("U", [0, 4])
@pytest.mark.parametrize("mode", ["argmax", "sampling"])
@pytest.mark.parametrize("rebase", [False, True])
def test_pool_schedule_reproduces_one_shot(ks, U, mode, rebase, monkeypatch):
    cfg = O.Config(32, 5, 8, 12, 3, 2, ks, U)
    p = O.make_params(cfg, 7 * ks + U)
    streams = _streams(cfg, 12, 3 * ks + U)
    if rebase:
        period = W.PoolSchedule(3, cfg.receptive_field, cfg.dilations, ks, U).period
        monkeypatch.setattr(W, "POOL_COUNTER_LIMIT", ks - 1 + period + 11)
    got, g0s, slots = _pool_run(cfg, p, streams, 3, mode, 5 * ks + U)
    for k, (x, total, h, uni, _) in enumerate(streams):
        want = O.batch_fast_generate(cfg, p, x[None], h[None], [total], mode, [uni])[0]
        assert got[k] == want.tolist(), k
    assert sum(len(v) for v in slots.values()) == len(streams) and len({s for v in slots.values() for s in v}) == 3
    assert all(b > a for a, b in zip(g0s, g0s[1:])) != rebase, g0s   # a rebase makes the counter go back


def test_schedule_rules():
    # rf 15 (ks 2, dilations 1 2 4 1 2 4), U 4: a one-sample seed needs frame 0 for sample 0
    dil = [1, 2, 4, 1, 2, 4]
    s = W.PoolSchedule(2, 15, dil, 2, 4)
    assert s.period == 4 and s.g == 1
    assert s.next_call() is None                            # nothing admitted
    a, b, c = s.add(0, 1, 10), s.add(1, 1, 3), s.add(2, 1, 5)
    assert s.next_call() is None                            # no frames: nobody runs, nobody is admitted
    b.frames = 1                                            # samples 0 .. 3 of b have their aux
    call = s.next_call()
    assert [st.sid for _, st, _, _ in call.rows] == [1] and call.n == 3 and call.g0 == 1 and call.finished == [1]
    assert [(T0, [st.sid for st in grp]) for T0, grp in call.admit] == [(1, [1])]
    a.frames, c.frames = 1, 3                               # a: 4 samples; c: complete
    call = s.next_call(max_samples=2)
    assert [(slot, st.sid, i0, n) for slot, st, i0, n in call.rows] == [(0, 0, 0, 2), (1, 2, 0, 2)] and call.g0 == 4
    call = s.next_call()                                    # a can run 2 more: the launch waits for it
    assert call.n == 2 and [n for _, _, _, n in call.rows] == [2, 2]
    assert s.next_call() is None                            # a starves: no launch, c waits too
    a.frames = 3                                            # complete: the longest remaining length bounds the call
    call = s.next_call()
    assert call.n == 6 and [(st.sid, n) for _, st, _, n in call.rows] == [(0, 6), (2, 1)] and call.finished == [0, 2]
    assert s.next_call() is None and not s.streams and s.finished == {0, 1, 2} and s.slots == [None, None]


def _fake(n):
    return [16 * (k + 1) for k in range(n)]   # non-NULL pointers: every check comes before any device work


def test_transplant_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    dil = (ctypes.c_int32 * 2)(1, 2)

    def call(src=16, src_B=4, rows=(0, 3), dst=32, cap=8, slots=(7, 0), rot=(-5, 9), n=2, R=512, ks=2, dl=dil, L=2):
        arr = lambda v: None if v is None else (ctypes.c_int32 * max(len(v), 1))(*v)
        return lib.wnb_decode_bf16_pool_transplant(src, src_B, arr(rows), dst, cap, arr(slots), arr(rot), n, R, ks, dl,
                                                   L, None)

    for kw in (dict(src_B=0), dict(cap=0), dict(n=0), dict(n=65), dict(R=0), dict(R=96), dict(ks=1), dict(L=0),
               dict(L=65)):
        assert call(**kw) == -1 and b"bad shape" in lib.wnb_last_error(), kw
    for kw in (dict(src=None), dict(dst=None), dict(rows=None), dict(slots=None), dict(rot=None), dict(dl=None)):
        assert call(**kw) == -1 and b"null pointer" in lib.wnb_last_error(), kw
    for kw in (dict(rows=(0, 4)), dict(rows=(-1, 0)), dict(slots=(8, 0)), dict(slots=(0, -1))):
        assert call(**kw) == -1 and b"source row" in lib.wnb_last_error(), kw
    assert call(slots=(3, 3)) == -1 and b"given twice" in lib.wnb_last_error()
    assert call(dl=(ctypes.c_int32 * 2)(1, 0)) == -1 and b"dilations must be positive" in lib.wnb_last_error()


def test_inputs_rejects_bad_arguments_without_gpu():
    lib = _lib.load()

    def call(ptrs=None, B=4, A=28, F=3, n=10, U=80):
        return lib.wnb_decode_bf16_pool_inputs(*(ptrs or _fake(6)), B, A, F, n, U, ctypes.c_uint64(1), None)

    for kw in (dict(B=0), dict(A=0), dict(F=0), dict(n=0), dict(U=-1)):
        assert call(**kw) == -1 and b"bad shape" in lib.wnb_last_error(), kw
    for i in (0, 3, 4):   # frames, table, aux (uniforms may be NULL: argmax)
        ptrs = _fake(6)
        ptrs[i] = None
        assert call(ptrs) == -1 and b"null pointer" in lib.wnb_last_error(), i
    for i in (1, 2):
        ptrs = _fake(6)
        ptrs[i] = None
        assert call(ptrs) == -1 and b"upsampling" in lib.wnb_last_error(), i


def test_pool_kernels_compile_without_spills():
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "decode_bf16_pool.cu"),
                            "-o", os.path.join(tmp, "d.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    assert not [line for line in text.splitlines() if "C7510" in line or "C7513" in line], text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, re.S):
        found[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert sorted(k for k in found if "pool_" in k) == sorted(found) and len(found) == 2, found
    assert all(v == (0, 0) for v in found.values()), found
