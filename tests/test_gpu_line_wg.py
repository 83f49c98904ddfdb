"""The line-graph kernels (launch_line_fwd / _bwd) at the tile counts their warpgroup layout makes special, through
tests/kernel_shim.cu against the float64 restatement in tests/kernel_units_ref.py.

The forward and the angle-update backward split the angles into 64-row tiles, and warpgroup w of CTA c owns the tiles
WG c + w, WG c + w + WG grid, ... with grid = min(ceil(tiles / WG), num_sms): WG = 3 in the angle-update forward
(k_line_fwd<false>), WG = 2 in the bond-conv forward (k_line_fwd<true>) and the angle-update backward
(k_line_bwd<false>).  The bond-conv backward keeps 128-row tiles, one per CTA.  The cases below put the partial last
tile on each warpgroup, leave the last CTA's later warpgroups without a tile, and make the warpgroups of one CTA loop a
different number of times, at one to three CTAs and at the device's SM count, with fewer angles than one tile among
them; rows that no angle maps to, and the padding rows of ang_out and gang, must keep their prefills bit for bit.

The CPU-only test at the end checks what the layout needs from the compiler: no spills in any fused tile kernel, and
the three-warpgroup forward within the 168 registers per thread that 384 threads on one SM leave.
"""
import os
import re
import subprocess

import pytest
import torch

from distmlip_b200 import build
from tests import kernel_units_ref as R

ERRS = {}
TW = 64  # angles per warpgroup tile


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = R.Shim(R.build_shim(tmp_path_factory.mktemp("kernel_shim")))
    yield s
    for k in sorted(ERRS):
        print(f"line max |out - ref| / scale  {k:<22s} {ERRS[k]:.3e}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles_per_warpgroup(A, num_sms, wg):
    """the number of 64-row tiles each warpgroup of each CTA runs, [grid][wg]"""
    ntiles = -(-A // TW)
    grid = min(-(-ntiles // wg), num_sms)
    return [[len(range(wg * c + w, ntiles, wg * grid)) for w in range(wg)] for c in range(grid)]


def layouts(A, hidden, num_sms):
    """{kernel: tiles per warpgroup} of the launches of a case that use the warpgroup layout"""
    if hidden:
        return {"fwd<H>": tiles_per_warpgroup(A, num_sms, 2)}
    return {"fwd<!H>": tiles_per_warpgroup(A, num_sms, 3), "bwd<!H>": tiles_per_warpgroup(A, num_sms, 2)}


def run_line(shim, c, ref, num_sms, what):
    A, hidden = c["A"], c["hidden"]
    dev = R.to_device(c, shim, "line")
    tag = "H" if hidden else "!H"
    if hidden:
        shim.line(False, True, c, dev, num_sms)
        torch.cuda.synchronize()
        R.check(ERRS, "line_fwd<H> aggB", R.TOL["line_fwd"], dev["aggB"], ref["aggB"], what)
        R.untouched("aggB", dev["aggB"], c["aggB"], c["a_out"], what)
    else:
        dev["ang_out"] = torch.full_like(dev["ang"], R.SENTINEL)
        shim.line(False, False, c, dev, num_sms)
        torch.cuda.synchronize()
        R.check(ERRS, "line_fwd<!H> ang_out", R.TOL["line_fwd"], dev["ang_out"][:A], ref["ang_out"][:A], what)
        assert bool((dev["ang_out"][A:] == R.SENTINEL).all()), f"ang_out padding rows written {what}"
    shim.line(True, hidden, c, dev, num_sms)
    torch.cuda.synchronize()
    R.check(ERRS, f"line_bwd<{tag}> gang", R.TOL["line_bwd"], dev["gang"][:A], ref["gang"][:A], what)
    assert bool(torch.isnan(dev["gang"][A:]).all()), f"gang padding rows touched {what}"
    for k, idx in (("gHa", "a_in"), ("gHb", "a_out"), ("gXc", "a_ctr")):
        R.check(ERRS, f"line_bwd<{tag}> {k}", R.TOL["line_bwd"], dev[k], ref[k], what)
        R.untouched(k, dev[k], c[k], c[idx], what)


def case(A, hidden, seed):
    c = R.gen_line(A, hidden, "random", seed)
    scales = R.line_scales(c)
    return c, {k: R.Mag(v, scales[k].s) for k, v in R.line_ref(c).items()}


# A: fewer angles than one tile (every warpgroup but the first idle); 2 tiles, the partial one on warpgroup 1; 3 tiles
# (three warpgroups: the partial tile on warpgroup 2; two: on warpgroup 0, whose partner idles at num_sms >= 2 and at
# one CTA runs one tile less); 4 and 5 tiles (the last CTA's later warpgroups idle, or at one CTA the first warpgroups
# run one tile more); every tile full (6 tiles); 11 and 13 tiles, so that each warpgroup loops
COUNTS = [5, TW + 30, 2 * TW + 30, 3 * TW + 1, 4 * TW + 63, 6 * TW, 10 * TW + 17, 12 * TW + 5]


@pytest.mark.gpu
@pytest.mark.parametrize("hidden", [True, False], ids=["H", "notH"])
@pytest.mark.parametrize("A", COUNTS)
def test_line_warpgroup_tiles(shim, A, hidden):
    c, ref = case(A, hidden, seed=200 + A)
    for num_sms in (1, 2, 3):
        run_line(shim, c, ref, num_sms, f"A={A} num_sms={num_sms} tiles={layouts(A, hidden, num_sms)}")


@pytest.mark.gpu
@pytest.mark.parametrize("hidden", [True, False], ids=["H", "notH"])
@pytest.mark.parametrize("extra", [5, TW + 5], ids=["wg0_one_more", "two_loop_more"])
def test_line_at_sm_count(shim, extra, hidden):
    # one full round of tiles on every warpgroup of every CTA (two rounds for the two-warpgroup backward of the angle
    # update), plus one or two tiles: extra = 5 gives warpgroup 0 of CTA 0 one tile more than warpgroup 1 in every
    # warpgroup kernel of the case; extra = TW + 5 gives it to warpgroups 0 and 1, the partial last tile on warpgroup 1
    A = (2 if hidden else 6) * TW * sms() + extra
    tiles = layouts(A, hidden, sms())
    for k, t in tiles.items():
        assert len(t) == sms(), k
        assert t[0][0] == t[0][1] + 1 if extra == 5 else t[0][0] == t[0][1], (k, t[0])
    c, ref = case(A, hidden, seed=11 + extra)
    run_line(shim, c, ref, sms(), f"A={A} num_sms={sms()}")


# ------------------------------------------------------------------------------------------------ ptxas, CPU only
def nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        return None


@pytest.mark.skipif(nvcc() is None, reason="nvcc not found")
def test_line_kernels_registers(tmp_path):
    out = subprocess.run([nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "kernels.cu"),
                                                      "-o", str(tmp_path / "kernels.o")],
                         cwd=build.CSRC, capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", out)
    line = {name: (int(st), int(ld), int(regs)) for name, st, ld, regs in props if "k_line_" in name}
    assert len(line) == 4, out
    assert not [k for k, v in line.items() if v[0] or v[1]], line
    fwd_angle = [v for k, v in line.items() if "k_line_fwdILb0E" in k]
    assert len(fwd_angle) == 1 and fwd_angle[0][2] <= 168, line
