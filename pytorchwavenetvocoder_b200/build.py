# -*- coding: utf-8 -*-
"""Build libwnb200.so (hand-written sm_90a kernels for the H100 + C ABI) in-tree with nvcc.

    python -m pytorchwavenetvocoder_b200.build [--force]

The library is a plain C-ABI shared object (no torch headers); cudart is linked statically and the
driver API (TMA descriptor encoding) is resolved at run time through cudaGetDriverEntryPoint, so the
.so loads on a machine without a GPU (CPU test tier).

Debugging builds: adding "-DWNB_WAIT_PRINTF" to NVCC_FLAGS makes a bounded mbarrier wait that times out (csrc/tc_ptx.cuh)
print its block and thread before it traps.  It is off by default because the printf call serialises every wgmma of the
tensor-core kernels (ptxas note C7510; tests/test_wgmma_pipeline.py checks that the default build has none).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libwnb200.so")
SOURCES = ["elementwise.cu", "resblock_simt.cu", "decode.cu", "decode_stream.cu", "decode_stream_prefill.cu", "wgrad_tc.cu", "decode_warp.cu", "decode_bf16.cu", "decode_prefill.cu", "decode_bf16_prefill.cu", "decode_bf16_pool.cu", "decode_bf16_park.cu", "decode_pool.cu", "gemm_nt_tc.cu", "resblock_z.cu", "stack.cu", "pack.cu", "loader.cu", "mlsa.cu", "melspc.cu", "melspc_stream.cu", "mcep.cu", "adam.cu", "score.cu", "distortion.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--fmad=true", "-cudart", "static"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "wnb200.h"),
                                                                os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, pr in procs:
        out = pr.communicate()[0].decode()
        if pr.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
        if verbose:
            print(out)
    cmd = [_nvcc(), "-shared", "-o", LIB, "-cudart", "static", "-Xcompiler", "-fPIC"] + objs + ["-ldl", "-lpthread", "-lrt"]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if out.returncode != 0:
        raise RuntimeError("link failed:\n%s" % out.stdout.decode())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
