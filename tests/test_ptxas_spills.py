"""The fused tile kernels (kernels.cu: k_atomconv_*, k_line_*) run one 256-thread CTA per SM close to the register
limit; a spill to local memory puts a round trip to L1 / L2 into their per-element loops.  Compiles kernels.cu for
sm_90a with the flags of the package build and `-Xptxas -v`, and fails if ptxas reports spill stores or loads in any
of them.  Needs nvcc, not a GPU.
"""
import os
import re
import subprocess

import pytest

from distmlip_b200 import build

FUSED = re.compile(r"k_atomconv_|k_line_")


def nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        return None


@pytest.mark.skipif(nvcc() is None, reason="nvcc not found")
def test_fused_tile_kernels_do_not_spill(tmp_path):
    out = subprocess.run([nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "kernels.cu"),
                                                      "-o", str(tmp_path / "kernels.o")],
                         cwd=build.CSRC, capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", out)
    fused = [(name, int(st), int(ld)) for name, st, ld in props if FUSED.search(name)]
    assert len(fused) == 6, out  # k_atomconv_fwd / _bwd, k_line_fwd / _bwd <true> / <false>
    spilled = [f for f in fused if f[1] or f[2]]
    assert not spilled, spilled
