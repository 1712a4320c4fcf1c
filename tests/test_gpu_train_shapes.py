# -*- coding: utf-8 -*-
"""GPU tier: the per-block tensor-core training path and the tensor-core post network against float64 across their
whole coverage, in tf32 and in bf16 (the table and what each row reaches: tests/train_shapes.py;
tests/test_train_shapes_host.py checks on the CPU that the rows reach every launch variant of the coverage grid).

* Block rows: every stage of one block -- z, xout, skip, z(bwd), dpre, dx, dhaux, dW1, db1, dW2, db2 -- teacher-forced
  against tests/tc_reference.py, inside sentinel margins, with NaN-filled outputs and nonzero gradient buffers
  (``_perblock`` of test_gpu_tc_stages.py with cv=to_tf32, ``_perblock_bf16`` of test_gpu_bf16.py with cv=to_bf16).
* Post rows: r1, logits, dh1, dskip, dWp1, dbp1, dWp2, dbp2 (``_post_stages`` of test_gpu_bf16.py), with the forward
  rectifying skip in place or taking it rectified.
* One training step of a whole model whose every block and post GEMM runs shapes no recipe has (Q 512, Ap 224, R 256,
  S 160, ks 3) against the float64 oracle, with the composed tf32 and the bf16 tolerances.
* A second backward of an R = 512, Ap = 224 row gives bit-identical gradients in each mode.

The largest err/bound of every stage is printed and, when $WNB_PARITY_OUT is set, written there (tc_stages_*.json)."""
import pytest

from oracle import wavenet_oracle as O
from tests import train_shapes as TS
from tests.test_bf16_host import to_bf16
from tests.test_gpu_bf16 import _oracle_case, _perblock_bf16, _post_stages
from tests.test_gpu_oracle_direct import TOL_COMPOSED, _dump, _summarise, _train_step_vs_oracle
from tests.tc_reference import to_tf32
from tests.test_gpu_tc_stages import _perblock

pytestmark = pytest.mark.gpu

BLOCK_CASES = [(rid, m) for rid, row in TS.BLOCK_ROWS.items() for m in row["modes"]]
POST_CASES = [(rid, m) for rid, row in TS.POST_ROWS.items() for m in row["modes"]]


def _run_block(rid, mode, repeat_bwd=False):
    row = TS.BLOCK_ROWS[rid]
    args = (row["R"], row["S"], row["Ap"], row["ks"], row["d"], row["B"], row["T"], row["last"], row["init"])
    seed = 7000 + list(TS.BLOCK_ROWS).index(rid)
    if mode == "tf32":
        assert _perblock(*args, seed=seed, repeat_bwd=repeat_bwd) == 2, rid     # the composed forward
    else:
        _perblock_bf16(*args, seed=seed, repeat_bwd=repeat_bwd)


@pytest.mark.parametrize("rid,mode", BLOCK_CASES, ids=["%s-%s" % c for c in BLOCK_CASES])
def test_block_row_stages(rid, mode):
    _run_block(rid, mode)


@pytest.mark.parametrize("rid,mode", POST_CASES, ids=["%s-%s" % c for c in POST_CASES])
def test_post_row_stages(rid, mode):
    row = TS.POST_ROWS[rid]
    S, Q, B, T = row["S"], row["Q"], row["B"], row["T"]
    _post_stages(S, Q, B, T, mode, to_tf32 if mode == "tf32" else to_bf16, row["rectified"],
                 9000 + list(TS.POST_ROWS).index(rid),
                 "%s_post_S%d_Q%d_B%d_T%d_rect%d" % (mode, S, Q, B, T, row["rectified"]))


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
def test_block_backward_is_deterministic(mode):
    """R = 512, Ap = 224: dW1's haux columns with nB 1 x n_split 7 beside 8 M-blocks in two launches"""
    rid = "r512_s160_a224_k2"
    assert TS.BLOCK_ROWS[rid]["R"] == 512 and TS.BLOCK_ROWS[rid]["Ap"] == 224
    _run_block(rid, mode, repeat_bwd=True)


# a model whose every launch takes a shape no recipe has: Q 512 (the N = 512 logits GEMM, 4 dWp2 M-blocks), n_aux 200
# (Ap 224: dhaux N 224, dW1 aux nB 1 x 7), R 256 (two gate launches of 128), S 160 (skip N 160, dWp1 nB 1 x 5), ks 3
_MODEL = O.Config(512, 200, 256, 160, 3, 2, 3, 0)


def test_model_step_tf32_vs_fp64_oracle():
    cfg = _MODEL
    rep = _summarise(_train_step_vs_oracle(cfg, 21, 2, 300, cfg.receptive_field, "tf32", False))
    _dump("parity_train_shapes_model_tf32.json", rep)
    print("composed tf32 (Q 512, Ap 224, R 256, S 160, ks 3) vs fp64 oracle: loss err %.2e, logits max err %.2e, "
          "worst weight %s %.3e, worst bias %s %.3e" % (rep["loss_abs_err"], rep["logits_max_abs_err"],
                                                       rep["worst_weight"][0], rep["worst_weight"][1],
                                                       rep["worst_bias"][0], rep["worst_bias"][1]))
    assert rep["loss_abs_err"] < TOL_COMPOSED["loss"], rep["loss_abs_err"]
    assert rep["logits_max_abs_err"] < TOL_COMPOSED["logits"], rep["logits_max_abs_err"]
    for k, v in rep["grads"].items():
        if v is None or v["numel"] == 1:
            continue
        tol = TOL_COMPOSED["weight"] if k.endswith("weight") else TOL_COMPOSED["bias"]
        assert v["rel_fro"] <= tol, (k, v)


def test_model_step_bf16_vs_fp64_oracle():
    cfg = _MODEL
    _oracle_case(cfg, 22, 2, 300, cfg.receptive_field, "train_shapes_model")
