"""The MACE kernels keep their per-thread state in registers: the message kernels hold a (atom, channel)'s accumulators
or adjoints and one edge's operands (up to 28 slots and 16 + 16 harmonics in the 0e+1o+2e reverse), split per output l
so that they fit (DESIGN.md §11.3).  Compiles kernels_mace.cu for sm_90a with the flags of the package build and
`-Xptxas -v`, and fails if ptxas reports spill stores or loads in any MACE kernel.  Needs nvcc, not a GPU.
"""
import os
import re
import subprocess

import pytest

from distmlip_b200 import build
from tests.test_ptxas_spills import nvcc


@pytest.mark.skipif(nvcc() is None, reason="nvcc not found")
def test_mace_kernels_do_not_spill(tmp_path):
    out = subprocess.run([nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "kernels_mace.cu"),
                                                      "-o", str(tmp_path / "kernels_mace.o")],
                         cwd=build.CSRC, capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", out)
    mace = [(name, int(st), int(ld)) for name, st, ld in props if "k_mace_" in name]
    l2 = [m for m in mace if "k_mace_msg_l2" in m[0]]
    assert len(l2) == 14, out  # forward and reverse, one per output l: 3 for max_ell 2, 4 for max_ell 3
    spilled = [m for m in mace if m[1] or m[2]]
    assert not spilled, spilled
