"""Build libb200mlip.so (sm_90a, H100) in-tree with nvcc.  `python -m distmlip_b200.build`.

The .so and the objects under csrc/build/ are build products (git-ignored); build() recompiles what is stale.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200mlip.so")
SOURCES = ["graph.cu", "kernels.cu", "kernels_wg.cu", "kernels_tn.cu", "kernels_mace.cu", "relax.cu", "engine.cu"]
HEADERS = ["common.cuh", "final_tail.cuh", "graph.cuh", "kernels.cuh", "wgmma.cuh", "engine_chgnet.inl", "tn_state.cuh", "engine_tn.inl", "mace_state.cuh", "mace_cg.cuh", "mace_cg_l2.cuh", "engine_mace.inl", "relax.cuh", os.path.join("..", "..", "include", "b200mlip.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--extended-lambda",
    "-Xcompiler", "-fPIC", "-Wno-deprecated-declarations",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = _nvcc()
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            subprocess.run(cmd, check=True, cwd=CSRC)
    if force or _stale(OUT, objs):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT] + objs + ["-ldl"]
        if verbose:
            print(" ".join(cmd))
        subprocess.run(cmd, check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
