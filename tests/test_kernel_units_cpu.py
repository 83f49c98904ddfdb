"""The kernel-unit tests (tests/test_gpu_kernel_units.py) without a GPU: the shim compiles and links against the built
library and its weight formatters run; the Mag restatement that carries the error scales computes the same values as
autograd; and the tolerances are sharp: on the inputs the GPU tests generate, every float64 mutant of an operation
(what a subtly wrong kernel would compute) exceeds the GPU tolerance by at least MUTANT_MARGIN on some element.
Needs nvcc for the shim, not a GPU.
"""
import pytest
import torch

from tests import kernel_units_ref as R
from tests.test_gpu_kernel_units import GEMM_M
from tests.test_ptxas_spills import nvcc

M_LONG = 6 * 128 + 45  # the run-pattern cases of the GPU tests


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    if nvcc() is None:
        pytest.skip("nvcc not found")
    return R.Shim(R.build_shim(tmp_path_factory.mktemp("kernel_shim")))


def test_shim_builds_and_formats_weights(shim):
    g = torch.Generator().manual_seed(0)
    raw = torch.randn(128, 64, generator=g)
    for img in (shim.second_layer_can(raw, False), shim.second_layer_can(raw, True), shim.line_reverse_can(raw)):
        assert img.numel() == 16384
    one = shim.canon_split(raw, 128, 64)
    hi, lo = one[:8192], one[8192:]
    assert torch.equal(hi, R.tf32(hi))
    assert torch.equal(torch.sort(hi.double() + lo.double()).values, torch.sort(raw.flatten().double()).values)
    rad = shim.radial_can(torch.randn(128, 9, generator=g), torch.randn(64, 9, generator=g))
    assert rad.numel() == shim.atom_rad
    with pytest.raises(RuntimeError, match="gemm_wg"):  # host-side argument checks come back as b2m errors
        shim.gemm_wg(None, 64, None, None, 64, 10, 64, 64, epi=1, stream=0)


@pytest.mark.parametrize("layer0", [True, False])
def test_atom_scales_carry_autograd_values(layer0):
    c = R.gen_atom(300, layer0, "random", seed=2)
    a, m = R.atom_ref(c), R.atom_scales(c)
    assert set(a) == set(m)
    for k, v in a.items():
        assert torch.allclose(v, m[k].x, rtol=1e-10, atol=1e-12), k
        assert bool((m[k].s >= v.abs() * (1 - 1e-12)).all()), k


@pytest.mark.parametrize("hidden", [True, False])
def test_line_scales_carry_autograd_values(hidden):
    c = R.gen_line(300, hidden, "random", seed=2)
    a, m = R.line_ref(c), R.line_scales(c)
    assert set(a) == set(m)
    for k, v in a.items():
        n = c["A"] if k in ("gang", "ang_out") else len(v)
        assert torch.allclose(v[:n], m[k].x[:n], rtol=1e-10, atol=1e-12), k


def assert_mutants_sharp(kind, c, tol_fwd, tol_bwd, expect):
    ref = R.atom_ref(c) if kind == "atom" else R.line_ref(c)
    sc = R.atom_scales(c) if kind == "atom" else R.line_scales(c)
    n = c["E"] if kind == "atom" else c["A"]
    for k in sc:  # padding rows of the angle buffers carry no reference
        if k in ("gang", "ang_out"):
            ref[k], sc[k] = ref[k][:n], R.Mag(sc[k].x[:n], sc[k].s[:n])
    fwd = {"agg", "aggB", "ang_out"}
    muts = R.mutants(kind, c)
    assert expect <= set(muts), (expect, set(muts))
    weak = {}
    for name, mut in muts.items():
        for k in ("gang", "ang_out"):
            if k in mut:
                mut[k] = mut[k][:n]
        # a mutant is caught if some output of the launch exceeds its tolerance by the margin
        ratio = max(R.max_err(torch.nan_to_num(mut[k], nan=0.0) if k in ("gang", "ang_out") else mut[k], ref[k],
                              sc[k].s) / (tol_fwd if k in fwd else tol_bwd) for k in ref)
        if ratio < R.MUTANT_MARGIN:
            weak[name] = ratio
    assert not weak, weak


@pytest.mark.parametrize("layer0", [True, False])
def test_atomconv_mutants_exceed_tolerance(layer0):
    # the GPU tests' run-pattern case with a run across tile boundaries and a partial last tile of 45 rows ...
    c = R.gen_atom(M_LONG, layer0, "long", seed=31)
    assert_mutants_sharp("atom", c, R.TOL["atom_fwd"], R.TOL["atom_bwd"],
                         {"tf32_W2", "tf32_radial", "no_be8", "no_b2_gate", "gd_no_M", "swap_dsig",
                          "run_head_before_tile_edge"})
    # ... and the count case whose last tile has 127 rows (rows 64..127 of it valid)
    c = R.gen_atom(5 * 128 + 127, layer0, "random", seed=5 * 128 + 127)
    assert_mutants_sharp("atom", c, R.TOL["atom_fwd"], R.TOL["atom_bwd"], {"rows_64_127_of_last_tile"})


@pytest.mark.parametrize("hidden", [True, False])
def test_line_mutants_exceed_tolerance(hidden):
    c = R.gen_line(M_LONG, hidden, "long", seed=17)
    expect = {"tf32_Wg", "swap_dsig", "run_head_before_tile_edge"} | ({"tf32_W2", "no_b2_gate"} if hidden else set())
    assert_mutants_sharp("line", c, R.TOL["line_fwd"], R.TOL["line_bwd"], expect)
    A = 5 * 128 + 127
    c = R.gen_line(A, hidden, "random", seed=A + 1)
    assert_mutants_sharp("line", c, R.TOL["line_fwd"], R.TOL["line_bwd"], {"rows_64_127_of_last_tile"})


@pytest.mark.parametrize("K,N", [(64, 128), (64, 64), (128, 64)])
def test_gemm_mutants_exceed_tolerance(K, N):
    tol = R.TOL["gemm"]
    for epi in (0, 1, 2):  # the operands of test_gemm_wg_shapes_sizes_flags, every flag set
        err = 0.0
        for M in GEMM_M:
            case = R.gen_gemm(M, K, N, seed=1000 * K + 10 * N + epi + M)
            ref, _ = R.gemm_ref(case["A"], case["W"], case["bias"], case["R"], case["Cold"], True, epi, case["Pre"])
            err = max(err, R.max_err(R.gemm_mutant(case, K, N, epi, (True, True, True)), ref.x, ref.s))
        assert err > R.MUTANT_MARGIN * tol, ("tf32 W", epi, err)
    M = 257
    for cross in ("lo_hi", "hi_lo"):
        case = R.gen_gemm(M, K, N, seed=5, cross=cross)
        ref, _ = R.gemm_ref(case["A"], case["W"])
        err = R.max_err(R.gemm_cross_mutant(case, cross), ref.x, ref.s)
        assert err > R.MUTANT_MARGIN * tol, (cross, err)
