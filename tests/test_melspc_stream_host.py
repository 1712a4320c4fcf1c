# -*- coding: utf-8 -*-
"""CPU tier: the host side of streaming mel-spectrogram extraction (wnb_melspc_stream, utils/melspc.py MelspcStream).

* ``melspc_frames_ready`` and ``melspc_carry_start`` against a brute force over ``reflect_index``: for every n and every
  later end length, the ready frames read only known samples and read the same ones whatever the end, and the pending
  frames read nothing before the carry start, which keeps fewer than fftl samples;
* a numpy executor of ``melspc_stream_plan`` (the two kernels restated over the same segment table and state layout),
  fed random chunkings, reproduces tests/melspc_reference.py's whole-signal filter, frames and features exactly;
* the state size, the argument checks made before any device work, MelspcStream's key bookkeeping (empty chunks launch
  nothing) and the ptxas register and spill counts of the stream kernels and of the whole-file kernels they share code
  with."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from pytorchwavenetvocoder_b200 import _lib, build
from pytorchwavenetvocoder_b200.utils import melspc as M
from tests import melspc_reference as R


# ---- the two rules ---------------------------------------------------------------------------------------------------
def _frame_idx(n_final, fftl, hop):
    """(frames, fftl) signal indices every frame of a signal of length n_final reads."""
    half = fftl // 2
    t = np.arange(1 + n_final // hop)[:, None]
    return M.reflect_index(t * hop - half + np.arange(fftl)[None, :], n_final)


def _check_rules(fftl, hop, n_max):
    """Every n <= n_max against every end length N in [n, n_max + fftl + hop)."""
    n_end = n_max + fftl + hop
    idx = {N: _frame_idx(N, fftl, hop) for N in range(1, n_end)}
    prev_cs = 0
    for n in range(1, n_max + 1):
        r = M.melspc_frames_ready(n, fftl, hop)
        cs = M.melspc_carry_start(n, fftl, hop)
        assert 0 <= n - cs < fftl, (fftl, hop, n, cs)      # fewer than fftl samples kept
        assert cs >= prev_cs, (fftl, hop, n)               # the carry only moves forward
        prev_cs = cs
        ref = idx[n][:r]
        assert ref.size == 0 or ref.max() < n              # ready frames read known samples only
        nexts = set()
        for N in range(n, n_end):
            I = idx[N]
            assert I.shape[0] >= r and np.array_equal(I[:r], ref), (fftl, hop, n, N)   # whatever the end
            assert not (I[r:] < cs).any(), (fftl, hop, n, N)                          # pending: nothing before cs
            nexts.add(I[r].tobytes() if I.shape[0] > r and I[r].max() < n else None)
        # frame r is not ready: some end drops it, makes it read an unknown sample, or changes what it reads
        assert None in nexts or len(nexts) > 1, (fftl, hop, n)


@pytest.mark.parametrize("fftl", [4, 6, 8, 12, 16])
def test_rules_brute_force_small(fftl):
    for hop in range(1, 12):
        _check_rules(fftl, hop, 4 * fftl)


@pytest.mark.parametrize("fftl,hops", [(32, [1, 5, 15, 16, 17, 40]), (64, [7, 31, 32, 33, 64, 80])])
def test_rules_brute_force_large(fftl, hops):
    for hop in hops:
        _check_rules(fftl, hop, 4 * fftl)


# ---- numpy executor of the plan --------------------------------------------------------------------------------------
class _NumpyStream(object):
    """The two kernels of csrc/melspc_stream.cu over melspc_stream_plan's table, in numpy: the FIR over
    [history | chunk] as tests/melspc_reference.py's ascending-tap sum, the frame windows through reflect_index over
    the scratch region [old carry | filtered chunk | new history], and the slot stores from scratch."""

    def __init__(self, fftl, hop, taps):
        self.fftl, self.hop, self.taps = fftl, hop, taps
        self.n_taps = 0 if taps is None else len(taps)
        self.H = max(self.n_taps - 1, 0)
        self.states = {}
        self.count = {}

    def push(self, chunks, final=()):
        keys = list(chunks) + [k for k in final if k not in chunks]
        segs = []
        for i, k in enumerate(keys):
            new = k not in self.count
            if new:
                self.count[k] = 0
                self.states[k] = np.full(self.H + self.fftl - 1, np.nan)   # never read before it is written
            segs.append((i, self.count[k], len(chunks.get(k, ())), k in final))
        tab, rows, scratch_n = M.melspc_stream_plan(segs, self.fftl, self.hop, self.n_taps)
        x = np.concatenate([np.asarray(chunks[k], dtype=np.float64) for k in keys if k in chunks] or [np.zeros(0)])
        scratch = np.full(scratch_n, np.nan)
        # launch 1: reads slots, writes scratch
        for u, k in enumerate(keys):
            d = tab[u]
            if not (d[M.SEG_R1] > d[M.SEG_R0] or d[M.SEG_FLAGS] & M.SEG_STORE):
                continue
            st = self.states[k]
            fresh = bool(d[M.SEG_FLAGS] & M.SEG_NEW)
            m, c, so = int(d[M.SEG_X_LEN]), int(d[M.SEG_N_BEFORE] - d[M.SEG_CARRY0]), int(d[M.SEG_SCRATCH])
            hist = np.zeros(self.H) if fresh else st[:self.H]
            comb = np.concatenate([hist, x[d[M.SEG_X_OFF]:d[M.SEG_X_OFF] + m]])
            scratch[so:so + c] = st[self.H:self.H + c]
            if self.n_taps:
                y = np.zeros(m)
                for kk, b in enumerate(self.taps):
                    y += b * comb[self.H - kk:self.H - kk + m]
            else:
                y = comb[self.H:]
            scratch[so + c:so + c + m] = y
            if d[M.SEG_FLAGS] & M.SEG_STORE:
                scratch[so + c + m:so + c + m + self.H] = comb[len(comb) - self.H:]
        # launch 2: reads scratch, writes frames and slots
        out = {}
        for u, k in enumerate(keys):
            d = tab[u]
            m, c, so = int(d[M.SEG_X_LEN]), int(d[M.SEG_N_BEFORE] - d[M.SEG_CARRY0]), int(d[M.SEG_SCRATCH])
            n_cur = int(d[M.SEG_N_BEFORE]) + m
            t = np.arange(d[M.SEG_R0], d[M.SEG_R1])[:, None]
            j = M.reflect_index(t * self.hop - self.fftl // 2 + np.arange(self.fftl)[None, :], n_cur) - d[M.SEG_CARRY0]
            assert j.size == 0 or (j.min() >= 0 and j.max() < c + m), (k, d)
            win = scratch[so + j]
            assert not np.isnan(win).any()
            out[k] = win
            if d[M.SEG_FLAGS] & M.SEG_STORE:
                st = self.states[k]
                st[:self.H] = scratch[so + c + m:so + c + m + self.H]
                keep0, keep = int(d[M.SEG_CARRY1] - d[M.SEG_CARRY0]), int(n_cur - d[M.SEG_CARRY1])
                st[self.H:self.H + keep] = scratch[so + keep0:so + keep0 + keep]
            self.count[k] = n_cur
        for k in final:
            del self.count[k], self.states[k]
        return out


def _chunking(n, fftl, hop, rng, kind):
    half = fftl // 2
    sizes = {"one": [1], "hop-1": [max(hop - 1, 0)], "hop+1": [hop + 1], "half": [half], "half+1": [half + 1],
             "fftl": [fftl], "zeros": [0, 1, 0, hop]}.get(kind)
    out, i = [], 0
    while i < n:
        s = int(rng.randint(0, 3 * fftl)) if sizes is None else sizes[len(out) % len(sizes)]
        out.append(min(s, n - i))
        i += out[-1]
    return out


@pytest.mark.parametrize("fftl,hop,cutoff", [(64, 80, 70), (64, 11, 0), (128, 40, 70), (256, 256, 70), (64, 32, 70)])
def test_numpy_executor_matches_whole_signal(fftl, hop, cutoff):
    fs = 16000
    taps = M.lowcut_taps(fs, cutoff) if cutoff else None
    rng = np.random.RandomState(fftl + hop + cutoff)
    half = fftl // 2
    basis = R.mel_basis(fs, fftl, 20, 0, fs // 2).astype(np.float64)
    for n in (1, 2, half, half + 1, fftl, 3 * fftl + 7, 700):
        x = rng.randint(-20000, 20000, n).astype(np.int16)
        whole_y = R.lowcut(x, taps)[0] if taps is not None else x.astype(np.float64)
        whole = R.frames(whole_y, fftl, hop)
        feats = R.melspc(x, fs, fftl, hop, 20, taps=taps)[0]
        for kind in ("one", "hop-1", "hop+1", "half", "half+1", "fftl", "zeros", "random", "random"):
            ex = _NumpyStream(fftl, hop, taps)
            sizes = _chunking(n, fftl, hop, rng, kind)
            got, i = [], 0
            for s_i, s in enumerate(sizes):
                last = s_i == len(sizes) - 1
                got.append(ex.push({"k": x[i:i + s]}, final=("k",) if last else ())["k"])
                i += s
            got = np.concatenate(got)
            assert np.array_equal(got, whole), (n, kind, sizes)
            mag = np.abs(np.fft.rfft(got / 32768 * R.hann(fftl), axis=1))
            assert np.array_equal(np.float32(np.log10(np.maximum(R.EPS, mag @ basis.T))), feats), (n, kind)


def test_numpy_executor_many_keys_and_reuse():
    """Keys of different lengths in one call, some with empty chunks, some ending early; new keys after others ended."""
    fftl, hop = 64, 13
    taps = M.lowcut_taps(16000, 70)
    rng = np.random.RandomState(5)
    sigs = {k: rng.randint(-3000, 3000, rng.randint(1, 500)).astype(np.int16) for k in range(12)}
    ex = _NumpyStream(fftl, hop, taps)
    pos = {k: 0 for k in sigs}
    got = {k: [] for k in sigs}
    live = set(range(6))
    nxt = 6
    while live:
        chunks, final = {}, []
        for k in sorted(live):
            s = int(rng.choice([0, 0, 1, hop, 40, 100]))
            chunks[k] = sigs[k][pos[k]:pos[k] + s]
            pos[k] += len(chunks[k])
            if pos[k] == len(sigs[k]) and rng.rand() < 0.5:
                final.append(k)
        for k, v in ex.push(chunks, final).items():
            got[k].append(v)
        for k in final:
            live.discard(k)
            if nxt < len(sigs):
                live.add(nxt)
                nxt += 1
    for k, x in sigs.items():
        assert np.array_equal(np.concatenate(got[k]), R.frames(R.lowcut(x, taps)[0], fftl, hop)), k


def test_plan_counts():
    tab, rows, scratch = M.melspc_stream_plan([(3, 0, 0, False), (1, 0, 600, False), (0, 600, 0, True)], 1024, 80, 255)
    assert rows == 0 + M.melspc_frames_ready(600, 1024, 80) + (1 + 600 // 80 - M.melspc_frames_ready(600, 1024, 80))
    assert list(tab[:, M.SEG_OUT_ROW]) == [0, 0, M.melspc_frames_ready(600, 1024, 80)]
    assert tab[0, M.SEG_FLAGS] == M.SEG_NEW and tab[1, M.SEG_FLAGS] == M.SEG_NEW | M.SEG_STORE
    assert tab[2, M.SEG_FLAGS] == 0 and list(tab[:, M.SEG_SLOT]) == [3, 1, 0]
    assert scratch == 600 + 254 + (600 - M.melspc_carry_start(600, 1024, 80))
    with pytest.raises(ValueError):
        M.melspc_stream_plan([(0, 0, 0, True)], 1024, 80, 255)


# ---- library entry points without a GPU --------------------------------------------------------------------------------
@pytest.mark.parametrize("fftl", [64, 1024, 4096])
@pytest.mark.parametrize("n_taps", [0, 1, 255, 1024])
def test_state_size(fftl, n_taps):
    lib = _lib.load()
    assert lib.wnb_melspc_stream_state_doubles(fftl, n_taps) == max(n_taps - 1, 0) + fftl - 1


@pytest.mark.parametrize("fftl,n_taps", [(32, 255), (8192, 255), (1000, 255), (1024, -1), (1024, 1025)])
def test_state_size_rejects(fftl, n_taps):
    assert _lib.load().wnb_melspc_stream_state_doubles(fftl, n_taps) == 0


def test_stream_rejects_bad_arguments():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)             # never dereferenced: every case fails before any device work

    def table(*rows):
        t = np.array(rows, dtype=np.int64).reshape(len(rows), M.SEG_FIELDS)
        return t

    good = M.melspc_stream_plan([(0, 0, 600, False), (1, 0, 10, True)], 1024, 80, 255)[0]

    def call(tab=good, n_frames=None, fftl=1024, hop=80, n_taps=255, n_slots=4, scratch=10 ** 6, mode=0, aux=None,
             mean=None, x=fake, states=fake):
        rows = int((tab[:, M.SEG_R1] - tab[:, M.SEG_R0]).sum()) if n_frames is None else n_frames
        return lib.wnb_melspc_stream(x, 1, len(tab), tab.ctypes.data_as(ctypes.c_void_p), fake, rows, fftl, hop, fake,
                                     n_taps, fake, fake, fake, fake, fake, 80, states, n_slots, fake, scratch, fake,
                                     mean, mean, mode, aux, None)

    def rejected(msg, rc=-1, **kw):
        assert call(**kw) == rc
        assert msg in lib.wnb_last_error(), lib.wnb_last_error()

    dup = good.copy()
    dup[1, M.SEG_SLOT] = 0
    rejected(b"slot 0 given twice", tab=dup)
    oob = good.copy()
    oob[1, M.SEG_SLOT] = 4
    rejected(b"slot 4 of 4", tab=oob)
    rejected(b"n_frames", n_frames=5)
    rejected(b"scratch", scratch=100)
    rejected(b"not supported", rc=-3, fftl=1000)
    rejected(b"not supported", rc=-3, fftl=8192)
    rejected(b"need hop > 0", hop=0)
    rejected(b"n_taps", n_taps=1025)
    rejected(b"scaler_mode", mode=1)
    rejected(b"needs mean and scale", aux=fake)
    rejected(b"null pointer", x=None)
    rejected(b"null pointer", states=None)
    carry = good.copy()
    carry[1, M.SEG_N_BEFORE] = 2000                # a carry longer than fftl - 1
    carry[1, M.SEG_FLAGS] = 0
    rejected(b"bad counts", tab=carry)
    frames = good.copy()
    frames[1, M.SEG_R1] += 5                       # more frames than the signal has
    rejected(b"bad frame range", tab=frames)
    big = M.melspc_stream_plan([(i, 0, 0, False) for i in range(1025)], 1024, 80, 255)[0]
    rejected(b"n_segs <= 1024", tab=big, n_slots=2000)


def test_stream_bookkeeping_without_gpu():
    s = M.MelspcStream(16000, 1024, 80, 80, highpass_cutoff=70, device="cpu")
    assert s.state_doubles == 254 + 1023
    e16 = torch.zeros(0, dtype=torch.int16)
    out = s.push({"a": e16, 7: e16, ("row", 2): e16})        # empty chunks: keys open, no launch
    assert set(out) == {"a", 7, ("row", 2)} and all(v.shape == (0, 80) for v in out.values())
    assert [s.slot(k) for k in ("a", 7, ("row", 2))] == [0, 1, 2]
    s.close(7)
    assert s.slot(7) is None
    with pytest.raises(KeyError):
        s.close(7)
    s.push({"b": e16, "c": e16})
    assert s.slot("b") == 1 and s.slot("c") == 3
    assert s.push({}) == {}
    for k in range(70):
        s.push({("n", k): torch.zeros(0, dtype=torch.float64)})
    assert sorted(s.slot(("n", k)) for k in range(70)) == list(range(4, 74))
    with pytest.raises(ValueError):
        s.push({}, final=["zz"])                               # a key that ends without a sample
    with pytest.raises(ValueError):
        s.push({"a": torch.zeros(0, dtype=torch.float32)})
    with pytest.raises(ValueError):
        s.push({"a": e16, "b": torch.zeros(0, dtype=torch.float64)})
    with pytest.raises(ValueError):
        s.push({"a": torch.zeros(2, 3, dtype=torch.int16)})
    with pytest.raises(_lib.WnbError):                         # samples on the CPU: no fallback
        s.push({"a": torch.zeros(5, dtype=torch.int16)})
    with pytest.raises(ValueError):
        M.MelspcStream(16000, 1000, 80, 80, device="cpu")
    with pytest.raises(ValueError):
        M.MelspcStream(16000, 1024, 80, 80, scaler=(np.zeros(79), np.ones(79)), device="cpu")
    sc = M.MelspcStream(16000, 1024, 80, 80, scaler=(np.zeros(80), np.ones(80)), device="cpu")
    assert sc.scaler_mode in (0, 2)
    assert sc.push({"a": e16})["a"].shape == (80, 0)


def _ptxas(src):
    nvcc = build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)):
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, src), "-o",
                            os.path.join(tmp, "k.cubin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = r.stdout.decode()
    assert r.returncode == 0, text
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", text, re.S):
        name = re.match(r"_ZN3wnb\d+(\w+?kernel)", m.group(1)).group(1)
        found[name] = (int(m.group(4)), int(m.group(2)), int(m.group(3)))
    return found


def test_ptxas_counts():
    assert "melspc_stream.cu" in build.SOURCES
    assert _ptxas("melspc_stream.cu") == {"stream_prep_kernel": (32, 0, 0), "stream_frames_kernel": (32, 0, 0)}
    assert _ptxas("melspc.cu") == {"melspc_kernel": (32, 0, 0), "lowcut_kernel": (32, 0, 0)}


# ---- bin/resynthesize.py: parser and refusals ----------------------------------------------------------------------------
def _conf(**kw):
    import argparse
    c = dict(n_quantize=256, n_aux=80, n_resch=64, n_skipch=64, dilation_depth=3, dilation_repeat=2, kernel_size=2,
             upsampling_factor=80, use_upsampling_layer=True, feature_type="melspc", use_speaker_code=False)
    c.update(kw)
    return argparse.Namespace(**c)


def test_cli_parser_defaults():
    from pytorchwavenetvocoder_b200.bin import feature_extract, resynthesize
    a = resynthesize.get_parser().parse_args(["--waveforms", "w", "--checkpoint", "c", "--outdir", "o", "--fmin", "",
                                              "--fmax", ""])
    f = feature_extract.get_parser().parse_args([])
    for k in ("shiftms", "fftl", "highpass_cutoff", "fs"):
        assert getattr(a, k) == getattr(f, k), k
    assert a.fmin is None and a.fmax is None and a.chunk_samples == 0 and a.batch_size == 32 and a.seed == 1
    assert a.decode_math == "fp32" and not a.noise_shaping


def test_cli_refusals():
    from pytorchwavenetvocoder_b200.bin.resynthesize import batches, check_setup
    ok = [("a.wav", (16000, 100))]
    assert check_setup(_conf(), (80,), 80, 16000, ok) == []
    cases = [(_conf(feature_type="world"), (80,), 80, ok, "feature_type 'world'"),
             (_conf(), (80,), 110, ok, "upsampling_factor 80"),
             (_conf(use_upsampling_layer=False), (80,), 80, ok, "no up-sampling layer"),
             (_conf(use_speaker_code=True), (80,), 80, ok, "speaker code"),
             (_conf(), (40,), 80, ok, "40 mel bands but the model's n_aux is 80"),
             (_conf(), (80,), 80, [("b.wav", (22050, 100))], "b.wav is sampled at 22050 Hz")]
    for conf, shape, hop, heads, msg in cases:
        errs = check_setup(conf, shape, hop, 16000, heads)
        assert len(errs) == 1 and msg in errs[0], (msg, errs)
    names = ["w%d" % i for i in range(7)]
    frames = [5, 3, 9, 3, 1, 7, 2]
    assert batches(names, frames, 1) == [[n] for n in names]
    order = [names[i] for i in np.argsort(frames)]
    assert sum(batches(names, frames, 3), []) == order and [len(b) for b in batches(names, frames, 3)] == [3, 2, 2]


def test_cli_exits_before_writing(tmp_path):
    from pytorchwavenetvocoder_b200.bin import resynthesize
    from pytorchwavenetvocoder_b200.utils import write_hdf5, write_wav_int16
    wavdir = tmp_path / "wav"
    wavdir.mkdir()
    write_wav_int16(str(wavdir / "a.wav"), 22050, np.zeros(500, dtype=np.int16))
    torch.save(_conf(), str(tmp_path / "model.conf"))
    write_hdf5(str(tmp_path / "stats.npz"), "/melspc/mean", np.zeros(80))
    out = tmp_path / "out"
    with pytest.raises(SystemExit) as e:
        resynthesize.main(["--waveforms", str(wavdir), "--checkpoint", str(tmp_path / "ck.pkl"), "--outdir", str(out),
                           "--stats", str(tmp_path / "stats.npz"), "--config", str(tmp_path / "model.conf")])
    assert e.value.code == 1 and not out.exists()
