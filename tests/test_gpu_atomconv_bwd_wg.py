"""The atom-conv backward (launch_atomconv_bwd) at the tile counts its warpgroup layout makes special, through
tests/kernel_shim.cu against the float64 restatement in tests/kernel_units_ref.py.

A CTA has two warpgroups, and warpgroup w of CTA c owns the 64-edge tiles 2 c + w, 2 c + w + 2 grid, ... with
grid = min(ceil(tiles / 2), num_sms).  The cases below put the partial last tile on either warpgroup, leave the last
CTA's second warpgroup without a tile, and make the two warpgroups of one CTA loop a different number of times, at one
to three CTAs and at the device's SM count; each runs in layer 0 (gA null: gC and gQ untouched) and in a later layer.
"""
import pytest
import torch

from tests import kernel_units_ref as R

pytestmark = pytest.mark.gpu
ERRS = {}
TW = 64  # edges per warpgroup tile


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = R.Shim(R.build_shim(tmp_path_factory.mktemp("kernel_shim")))
    yield s
    for k in sorted(ERRS):
        print(f"atomconv_bwd max |out - ref| / scale  {k:<22s} {ERRS[k]:.3e}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles_per_warpgroup(E, num_sms):
    """the number of tiles each warpgroup of each CTA runs, [grid][2]"""
    ntiles = -(-E // TW)
    grid = min(-(-ntiles // 2), num_sms)
    return [[len(range(2 * c + w, ntiles, 2 * grid)) for w in range(2)] for c in range(grid)]


def run_bwd(shim, c, ref, num_sms, what):
    dev = R.to_device(c, shim, "atom")
    for k in ("gC", "gQ", "gd", "gA"):
        dev[k] = c[k].to("cuda").clone()
    if c["layer0"]:
        dev["gA"] = None
    shim.atomconv(True, c, dev, num_sms)
    torch.cuda.synchronize()
    tol = R.TOL["atom_bwd"]
    R.check(ERRS, "atomconv_bwd gd", tol, dev["gd"], ref["gd"], what)
    if c["layer0"]:
        assert torch.equal(dev["gC"].cpu(), c["gC"]), f"gC written in layer 0 {what}"
        assert torch.equal(dev["gQ"].cpu(), c["gQ"]), f"gQ written in layer 0 {what}"
    else:
        R.check(ERRS, "atomconv_bwd gA", tol, dev["gA"], ref["gA"], what)
        R.check(ERRS, "atomconv_bwd gC", tol, dev["gC"], ref["gC"], what)
        R.check(ERRS, "atomconv_bwd gQ", tol, dev["gQ"][: c["B_own"]], ref["gQ"][: c["B_own"]], what)
        R.untouched("gA", dev["gA"], c["gA"], c["e_src"], what)
        R.untouched("gC", dev["gC"], c["gC"], c["e_dst"], what)


def case(E, layer0, seed):
    c = R.gen_atom(E, layer0, "random", seed)
    scales = R.atom_scales(c)
    return c, {k: R.Mag(v, scales[k].s) for k, v in R.atom_ref(c).items()}


# E: one partial tile (warpgroup 1 of the only CTA idle); the partial last tile on warpgroup 1 (2, 4 tiles) or on
# warpgroup 0 (3, 5 tiles: the last CTA's warpgroup 1 idle at num_sms >= 2, and at 2 / 1 CTAs warpgroup 0 runs one
# tile more than warpgroup 1); every tile full (6 tiles); 11 tiles, so that each warpgroup loops
COUNTS = [5, TW + 30, 2 * TW + 30, 3 * TW + 1, 4 * TW + 63, 6 * TW, 10 * TW + 17]


@pytest.mark.parametrize("layer0", [True, False], ids=["layer0", "layerN"])
@pytest.mark.parametrize("E", COUNTS)
def test_atomconv_bwd_warpgroup_tiles(shim, E, layer0):
    c, ref = case(E, layer0, seed=100 + E)
    for num_sms in (1, 2, 3):
        run_bwd(shim, c, ref, num_sms, f"E={E} num_sms={num_sms} tiles={tiles_per_warpgroup(E, num_sms)}")


@pytest.mark.parametrize("layer0", [True, False], ids=["layer0", "layerN"])
@pytest.mark.parametrize("extra", [5, TW + 5], ids=["wg0_one_more", "both_loop"])
def test_atomconv_bwd_at_sm_count(shim, extra, layer0):
    # extra = 5: warpgroup 0 of CTA 0 runs a second, partial tile and warpgroup 1 does not; extra = TW + 5: both
    # warpgroups of CTA 0 loop, the partial last tile on warpgroup 1
    E = 2 * TW * sms() + extra
    tiles = tiles_per_warpgroup(E, sms())
    assert len(tiles) == sms()
    if extra == 5:
        assert tiles[0] == [2, 1]
    else:
        assert tiles[0] == [2, 2]
    c, ref = case(E, layer0, seed=7 + extra)
    run_bwd(shim, c, ref, sms(), f"E={E} num_sms={sms()}")
