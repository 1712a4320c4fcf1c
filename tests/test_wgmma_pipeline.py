# -*- coding: utf-8 -*-
"""The tensor-core kernels keep their wgmma asynchronous: ptxas serialises every wgmma.mma_async of a kernel that makes
a function call (a device printf, say) inside its wgmma pipeline, and says so only in an informational note (C7510)
under -Xptxas -v.  Compile the three wgmma translation units for sm_90a and require that no such note appears and that
the gemm_nt_tc kernels do not spill.  Needs nvcc, not a GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from pytorchwavenetvocoder_b200 import build

UNITS = ["gemm_nt_tc.cu", "wgrad_tc.cu", "resblock_z.cu"]


def _nvcc():
    try:
        cand = build._nvcc()
    except RuntimeError:
        return None
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.fixture(scope="module")
def ptxas_reports():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for src in UNITS:
            cmd = [nvcc] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, src),
                                    "-o", os.path.join(tmp, src + ".cubin")]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        for src, pr in procs:
            text = pr.communicate()[0].decode()
            assert pr.returncode == 0, text
            out[src] = text
    return out


@pytest.mark.parametrize("src", UNITS)
def test_no_serialised_wgmma(ptxas_reports, src):
    notes = [line for line in ptxas_reports[src].splitlines() if "C7510" in line]
    assert not notes, "\n".join(notes)


def test_gemm_nt_tc_does_not_spill(ptxas_reports):
    spills = re.findall(r"Function properties for (\S*gemm_nt_tc_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                        r"stores", ptxas_reports["gemm_nt_tc.cu"])
    assert len(spills) == 40
    assert all(int(n) == 0 for _, n in spills), spills
