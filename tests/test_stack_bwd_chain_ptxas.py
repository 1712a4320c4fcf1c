# -*- coding: utf-8 -*-
"""The stack backward's block-boundary kernel (csrc/stack_bwd_chain.cu) keeps its wgmma asynchronous and its registers:
compile it for sm_90a with -Xptxas -v and require that both instantiations (with and without the dhaux output) exist, do
not spill, and draw none of the notes with which ptxas reports serialised wgmma (C7510, C7512, C7513) or a warpgroup
fence it had to inject between wgmma and the registers (C7519).  Needs nvcc, not a GPU."""
import os
import re
import subprocess
import tempfile

import pytest

from pytorchwavenetvocoder_b200 import build
from tests.test_wgmma_pipeline import _nvcc


@pytest.fixture(scope="module")
def report():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "stack_bwd_chain.cu"),
                                "-o", os.path.join(tmp, "chain.cubin")]
        pr = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    text = pr.stdout.decode()
    assert pr.returncode == 0, text
    return text


def test_chain_kernel_in_build():
    assert "stack_bwd_chain.cu" in build.SOURCES


def test_chain_kernel_does_not_spill(report):
    spills = re.findall(r"Function properties for (\S*stack_bwd_chain_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", report)
    assert len(spills) == 2, report
    assert all(int(s) == 0 and int(l) == 0 for _, s, l in spills), spills


def test_chain_kernel_wgmma_not_serialised(report):
    notes = [line for line in report.splitlines() if re.search(r"C751[0239]", line)]
    assert not notes, "\n".join(notes)
