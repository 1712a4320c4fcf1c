# -*- coding: utf-8 -*-
"""GPU tier: the tf32 deferred-skip stack and the fused R = 64 per-block path against float64 across their whole
coverage (the table and what each row reaches: tests/stack_shapes.py; tests/test_stack_shapes_host.py checks on the
CPU that the rows reach every launch variant of the coverage grid).

* Stack rows: every stage of ``wnb_stack_fwd`` / ``wnb_stack_bwd`` -- z, xout, skip, dZ_all, dpre, dx, dhaux, dW1,
  db1, dW2res, db2res, dWskip, dbskip, block by block -- teacher-forced against tests/tc_reference.py, inside sentinel
  margins, with NaN-filled outputs and nonzero gradient buffers (``_stack_stages`` of test_gpu_tc_stages.py, which
  runs the six cases of the table itself); rows with ``aux`` off pass dhaux = NULL.
* Fused rows: every stage of one block on ``resblock_fwd_skip`` and the R = 64 gate-GEMM backward (``_perblock``),
  with dhaux = NULL where ``aux`` is off.
* A second ``wnb_stack_bwd`` of the L = 59 row (three weight-gradient launches) gives bit-identical results.
* One row run in a child process whose kernels all walk their time tiles front to back (WNB_ALT_DIR=0) gives
  bit-identical results: the tile direction only reorders independent tiles.
* One training step against the float64 oracle of a U = 0 model on the stack (dhaux never computed) and of a model
  whose skip width only the fused path takes (S = 384).

The largest err/bound of every stage is printed and, when $WNB_PARITY_OUT is set, written there (tc_stages_*.json)."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import wavenet_oracle as O
from tests import stack_shapes as SS
from tests.test_gpu_oracle_direct import TOL_TF32, TOL_TF32_SAME_MASKS, _dump, _summarise, _train_step_vs_oracle
from tests.test_gpu_tc_stages import SENTINEL, _perblock, _stack_stages

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STACK_CASES = [rid for rid in SS.STACK_ROWS if not rid.startswith("case_")]   # the six run in test_gpu_tc_stages
FUSED_CASES = list(SS.FUSED_ROWS)


def _run_stack_row(rid, repeat_bwd=False, check=True):
    row = SS.STACK_ROWS[rid]
    L, S, B, T = row["L"], row["S"], row["B"], row["T"]
    seed = 11000 + list(SS.STACK_ROWS).index(rid)
    return _stack_stages(L, S, B, T, row["dilations"], row["relu"], row["aux"], seed,
                         "stack_row_%s_L%d_S%d_B%d_T%d" % (rid, L, S, B, T), repeat_bwd=repeat_bwd, check=check)


@pytest.mark.parametrize("rid", STACK_CASES)
def test_stack_row_stages(rid):
    _run_stack_row(rid)


@pytest.mark.parametrize("rid", FUSED_CASES)
def test_fused_row_stages(rid):
    row = SS.FUSED_ROWS[rid]
    assert _perblock(64, row["S"], 32, 2, row["d"], row["B"], row["T"], row["last"], row["init"],
                     seed=12000 + FUSED_CASES.index(rid), dhaux=row["aux"]) == 1, rid    # the fused forward


def test_stack_backward_is_deterministic():
    """353 weight-gradient problems in three launches: every output of a second backward is bit-identical"""
    rid = "l59_s512_aux"
    assert (SS.STACK_ROWS[rid]["L"], SS.STACK_ROWS[rid]["S"]) == (59, 512)
    _run_stack_row(rid, repeat_bwd=True, check=False)


_CHILD = """
import sys, torch
from tests import test_gpu_stack_shapes as M
out = M._run_stack_row(sys.argv[1], check=False)
torch.save({k: v.cpu() for k, v in out.items()}, sys.argv[2])
"""


def test_tile_direction_changes_no_bit(tmp_path):
    """The stack alternates the direction in which consecutive kernels walk their time tiles (for L2 reuse); the
    direction is read once per process, so the other setting runs in a child process, which exits before the test
    returns.  Every output, the workspace included, must be bit-identical."""
    rid = "l7_s192_aux"
    row = SS.STACK_ROWS[rid]
    assert row["L"] == 7 and row["aux"] and row["B"] * -(-row["T"] // 64) > 2
    here = _run_stack_row(rid, check=False)
    torch.cuda.synchronize()
    alt_here = not os.environ.get("WNB_ALT_DIR", "").startswith("0")
    env = dict(os.environ, WNB_ALT_DIR="0" if alt_here else "1")
    env["PYTHONPATH"] = ROOT + (os.pathsep + env["PYTHONPATH"] if env.get("PYTHONPATH") else "")
    path = str(tmp_path / "child.pt")
    flags = ["-s"] if sys.flags.no_user_site else []
    proc = subprocess.run([sys.executable] + flags + ["-c", _CHILD, rid, path], cwd=ROOT, env=env, timeout=600,
                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert proc.returncode == 0, proc.stdout.decode(errors="replace")[-4000:]
    there = torch.load(path)
    assert set(there) == set(here)
    for k, v in here.items():
        # (the workspace's never-written slots are NaN in both)
        assert torch.equal(v.cpu().nan_to_num(SENTINEL), there[k].nan_to_num(SENTINEL)), \
            "%s differs with the tile direction" % k


def _report_step(rep, what):
    print("%s vs fp64 oracle: loss err %.2e, logits max err %.2e, worst weight %s %.3e, worst bias %s %.3e"
          % (what, rep["loss_abs_err"], rep["logits_max_abs_err"], rep["worst_weight"][0], rep["worst_weight"][1],
             rep["worst_bias"][0], rep["worst_bias"][1]))
    if rep.get("worst_weight_same_masks"):
        print("   with the oracle's ReLU masks replaced by ours (flip fraction %s): worst weight %s %.3e, worst bias "
              "%s %.3e" % (rep["relu_mask_flip_fraction"], rep["worst_weight_same_masks"][0],
                        rep["worst_weight_same_masks"][1], rep["worst_bias_same_masks"][0],
                        rep["worst_bias_same_masks"][1]))


def _assert_step(rep, keys):
    assert rep["loss_abs_err"] < TOL_TF32["loss"], rep["loss_abs_err"]
    assert rep["logits_max_abs_err"] < TOL_TF32["logits"], rep["logits_max_abs_err"]
    for key, tols in keys:
        assert rep[key], key
        for k, v in rep[key].items():
            if v is None or v["numel"] == 1:
                continue
            tol = tols["weight"] if k.endswith("weight") else tols["bias"]
            assert v["rel_fro"] <= tol, (key, k, v)


def test_stack_model_without_upsampling_vs_fp64_oracle():
    """U = 0 (aux at the sample rate): the stack backward runs without dhaux -- the no-aux chain kernel and dx_0"""
    cfg = O.Config(256, 28, 64, 256, 10, 2, 2, 0)
    T = cfg.receptive_field + 553
    rep = _summarise(_train_step_vs_oracle(cfg, 31, 2, T, cfg.receptive_field, "tf32", True))
    _dump("parity_stack_shapes_u0_tf32.json", rep)
    _report_step(rep, "tf32 stack, U = 0 (64 res / 256 skip, 20 blocks)")
    _assert_step(rep, (("grads", TOL_TF32), ("grads_same_relu_masks", TOL_TF32_SAME_MASKS)))


def test_fused_only_model_vs_fp64_oracle():
    """S = 384: not a stack width, so every block runs the fused forward and the R = 64 gate-GEMM backward"""
    cfg = O.Config(256, 28, 64, 384, 10, 2, 2, 0)
    T = cfg.receptive_field + 553
    rep = _summarise(_train_step_vs_oracle(cfg, 32, 2, T, cfg.receptive_field, "tf32", False))
    _dump("parity_stack_shapes_fused_s384_tf32.json", rep)
    _report_step(rep, "tf32 fused per-block path (64 res / 384 skip, 20 blocks)")
    _assert_step(rep, (("grads", TOL_TF32),))
