# -*- coding: utf-8 -*-
"""GPU tier: the fp32 streaming and direct decoders against float64 across the shapes their launch rules cover, one row
per branch (the table and what each row reaches: tests/decode_shapes.py; tests/test_decode_shapes_host.py checks on
the CPU that each row reaches it).

* Rows the streaming rule covers run ``auto`` (the streaming decoder after its parallel warm-up) and ``direct`` by name;
  rows only the direct decoder covers run ``auto``, which must pick ``direct``, and ``kernel="stream"`` must raise.
  Every row runs argmax, supplied uniforms and in-kernel Philox.  Every step's logits are compared with the
  teacher-forced float64 forward and every pick must be admissible (``_check`` of test_gpu_decode_forms.py).
* Streaming rows: the parallel warm-up and the sequential warm-up give ``torch.equal`` codes, ``logits_out`` and queue
  workspace (``_paths`` of test_gpu_decode_stream_prefill.py).
* A direct-only row decoded as a session fed in random chunks is bit-identical to one-shot decoding.
* Shapes neither decoder covers raise ``WnbError`` and leave the process able to decode.

Bound.  Per row and mode, e32 is the worst |float32 teacher-forced forward - float64| over the same positions
(``forward64(dtype=torch.float32)`` on the GPU, TF32 off): what float32 evaluation alone costs at that shape.  The
kernel's worst |logit - float64| must be at most RATIO * e32 + ABS_FLOOR.  Each row's err/e32 is printed and, when
$WNB_PARITY_OUT is set, written there as decode_shapes_*.json.  A failure names the row, the utterance, the step and
the class.
"""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from tests import decode_reference as D
from tests import decode_shapes as T
from tests.test_gpu_decode_forms import _decode, _dump, _inputs, _nsm, _run_modes
from tests.test_gpu_decode_stream_prefill import _assert_equal, _paths
from tests.util import our_model

pytestmark = pytest.mark.gpu

RATIO = 4.0
ABS_FLOOR = 2.0 ** -22      # 2.4e-7: two float32 ulps of a logit of magnitude 1
T0 = 3                      # a seed shorter than every row's receptive field: n_pad > 0

_CACHE = {}


def _model(rid):
    """(cfg, net, p64) of a row, the row's dilations set on the oracle config and the model alike; one row cached"""
    if rid not in _CACHE:
        _CACHE.clear()
        row = T.ROWS[rid]
        cfg = O.Config(*row["shape"])
        cfg.dilations = T.dilations(row)
        cfg.receptive_field = (cfg.kernel_size - 1) * sum(cfg.dilations) + 1
        p = O.make_params(cfg, 500 + list(T.ROWS).index(rid))
        net = our_model(cfg, p).eval()
        net.dilations = list(cfg.dilations)   # the weights do not depend on the dilations
        net.receptive_field = cfg.receptive_field
        _CACHE[rid] = (cfg, net, {k: v.astype(np.float64) for k, v in p.items()})
    return _CACHE[rid]


@pytest.fixture
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _calibrate(cfg, p64, x, h, n_list):
    """on_mode hook of _run_modes: e32 over the positions compared, and where the kernel's worst error is"""
    def run(mode, gen, lg, ref):
        max_n = max(n_list)
        ref32 = D.teacher_forced_logits(cfg, p64, x, h, gen[:, :max_n], device="cuda", chunk=8, dtype=torch.float32)
        valid = np.arange(max_n)[None, :] < np.asarray(n_list)[:, None]
        e32 = float(np.abs(ref32 - ref).max(-1)[valid].max())
        err = np.abs(lg.astype(np.float64) - ref)
        err[~valid] = 0
        b, i, q = np.unravel_index(int(np.argmax(err)), err.shape)
        return {"e32": e32, "worst": {"utt": int(b), "step": int(i), "class": int(q), "got": float(lg[b, i, q]),
                                     "want": float(ref[b, i, q])}}
    return run


def _assert_rows(what, rows):
    for m, r in rows.items():
        assert not r["bad_picks"], ("%s %s: inadmissible picks (utt, step, class)" % (what, m),
                                    [(b["utt"], b["step"], b["pick"]) for b in r["bad_picks"]])
        w = r["worst"]
        assert r["max_err"] <= RATIO * r["e32"] + ABS_FLOOR, (
            "%s %s: |logit - float64| %.3e > %g * e32 (%.3e) + %.1e at utterance %d step %d class %d: %.9g against %.9g"
            % (what, m, r["max_err"], RATIO, r["e32"], ABS_FLOOR, w["utt"], w["step"], w["class"], w["got"], w["want"]))


def _vs_fp64(rid, kernel, expect):
    cfg, net, p64 = _model(rid)
    row = T.ROWS[rid]
    nsm = _nsm()
    report = {}
    for k, bfn in enumerate(row["batches"]):
        B = bfn(nsm)
        x, h, n_list = _inputs(cfg, B, T0, row["max_n"], 700 + k)
        rows = _run_modes(cfg, net, p64, x, h, n_list, kernel, 7000 + k, expect=expect,
                          on_mode=_calibrate(cfg, p64, x, h, n_list))
        report[B] = rows
        print("%s %s (ran %s) B=%d: err/e32 %s" % (rid, kernel, expect, B, {
            m: "%.2e/%.2e = %.2f" % (r["max_err"], r["e32"], r["max_err"] / max(r["e32"], 1e-30))
            for m, r in rows.items()}))
        _dump("decode_shapes_%s_%s_B%d.json" % (rid, kernel, B), {"row": rid, "kernel": kernel, "ran": expect, "B": B,
                                                                   "modes": rows, "ratio": RATIO})
    for B, rows in report.items():
        _assert_rows("row %s kernel %s B=%d" % (rid, kernel, B), rows)


STREAM_ROWS = [r for r, v in T.ROWS.items() if v["rule"] == "stream"]
DIRECT_ROWS = [r for r, v in T.ROWS.items() if v["rule"] == "direct"]


@pytest.mark.parametrize("rid,kernel", [(r, k) for r in STREAM_ROWS for k in ("auto", "direct")])
def test_streaming_rows_vs_fp64(rid, kernel, no_tf32):
    _vs_fp64(rid, kernel, "stream" if kernel == "auto" else "direct")


@pytest.mark.parametrize("rid", DIRECT_ROWS)
def test_direct_rows_vs_fp64(rid, no_tf32):
    from pytorchwavenetvocoder_b200 import _lib
    cfg, net, p64 = _model(rid)
    x, h, n_list = _inputs(cfg, 3, T0, 4, 1)
    with pytest.raises(_lib.WnbError):
        _decode(net, x, h, n_list, "argmax", "stream")
    _vs_fp64(rid, "auto", "direct")


@pytest.mark.parametrize("rid", STREAM_ROWS)
def test_streaming_rows_prefill_equals_sequential(rid):
    from tests.test_gpu_decode_stream_prefill import _inputs as stream_inputs
    _, net, _ = _model(rid)
    max_n = T.ROWS[rid]["max_n"]
    x, h, n_list = stream_inputs(net, 3, T0, max_n, 31)
    uni = torch.from_numpy(np.random.RandomState(32).uniform(size=(3, max_n)).astype(np.float32))
    _assert_equal(_paths(net, x, h, n_list, "argmax"), (rid, "argmax"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", uniforms=uni), (rid, "uniforms"))
    _assert_equal(_paths(net, x, h, n_list, "sampling", seed=4321), (rid, "philox"))


def test_direct_session_in_random_chunks_equals_one_shot():
    from pytorchwavenetvocoder_b200.nets.wavenet import DecodeSession
    _, net, _ = _model("odd_rs_q255")
    B, max_n, seed = 3, 40, 99
    rng = np.random.RandomState(5)
    x = torch.from_numpy(rng.randint(0, net.n_quantize, size=(B, T0))).cuda()
    h = torch.from_numpy(rng.standard_normal((B, net.n_aux, T0 + max_n + 1)).astype(np.float32)).cuda()
    n_list = [max_n, 1, 17]
    with torch.no_grad():
        want, want_lg = net._decode(x, h, n_list, "sampling", return_logits=True, seed=seed)
        assert net.last_decode_kernel == "direct"
        s = DecodeSession(net, x, n_list, "sampling", seed, None, True, "auto")
        assert s.kernel == "direct"
        codes, logits = [[] for _ in range(B)], [[] for _ in range(B)]
        f0 = 0
        while not s.done:
            F = int(rng.randint(1, 7))
            gen, lg = s.step(h[:, :, f0:f0 + F])
            f0 += F
            for b, c in enumerate(s.last_counts):
                codes[b].append(gen[b, :c].cpu())
                logits[b].append(lg[b, :c].cpu())
    for b, n in enumerate(n_list):
        assert torch.equal(torch.cat(codes[b]), want[b, :n].cpu()), b
        assert torch.equal(torch.cat(logits[b]), want_lg[b, :n].cpu()), b


@pytest.mark.parametrize("rid", [r for r, v in T.ROWS.items() if v["rule"] == "none"])
def test_uncovered_shape_raises_and_decoding_goes_on(rid):
    from pytorchwavenetvocoder_b200 import _lib
    cfg0, net0, _ = _model("d1")
    x0, h0, n0 = _inputs(cfg0, 3, T0, 8, 2)
    before = _decode(net0, x0, h0, n0, "sampling", "auto", seed=3, expect="direct")
    cfg, net, _ = _model(rid)
    x, h, n_list = _inputs(cfg, 3, T0, T.ROWS[rid]["max_n"], 3)
    for kernel in ("auto", "direct", "stream"):
        with pytest.raises(_lib.WnbError):
            with torch.no_grad():
                net._decode(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), n_list, "argmax", kernel=kernel)
    torch.cuda.synchronize()          # no sticky error
    cfg0, net0, _ = _model("d1")
    after = _decode(net0, x0, h0, n0, "sampling", "auto", seed=3, expect="direct")
    assert np.array_equal(before[0], after[0])
    for b, n in enumerate(n0):       # logits past an utterance's length are not written
        assert np.array_equal(before[1][b, :n], after[1][b, :n]), b
