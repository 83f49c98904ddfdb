"""The MACE kernel-unit tests (tests/test_gpu_mace_units.py) without a GPU: the shim's MACE host entries run the
engine's own conv-path list and symmetric-contraction term builder, which must reproduce tests/mace_eq_ref.py and the
float64 U contraction; the reverse walked over the shipped term list equals autograd of the contraction modules; every
scale bounds its value; and the tolerances are sharp: on inputs built as the GPU tests build them, every float64 mutant
(what a subtly wrong kernel or term builder would compute) exceeds its tolerance by at least MUTANT_MARGIN on some
element.  Needs nvcc for the shim, not a GPU.
"""
import pytest
import torch

from tests import kernel_units_ref as KU
from tests import mace_eq_ref as EQ
from tests import mace_units_ref as M
from tests.test_ptxas_spills import nvcc


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    if nvcc() is None:
        pytest.skip("nvcc not found")
    return KU.Shim(KU.build_shim(tmp_path_factory.mktemp("kernel_shim")))


RATIOS = {}


def ratio(name, tol, pairs):
    """largest over (mutant value, Mag ref) pairs of max |mut - ref| / scale / tol; recorded and printed"""
    r = max(KU.max_err(mut, ref.x, ref.s) for mut, ref in pairs) / M.TOL[tol]
    RATIOS[name] = min(RATIOS.get(name, float("inf")), r)
    print(f"mace mutant {name:<24s} {r:.3g} x tol")
    return r


def sharp(name, tol, pairs):
    r = ratio(name, tol, pairs)
    assert r >= KU.MUTANT_MARGIN, (name, r)


# ------------------------------------------------------------------------------------------------ host code
@pytest.mark.parametrize("hidden_l", [0, 1])
def test_conv_paths_match_oracle(shim, hidden_l):
    for max_ell in range(4):
        assert shim.mace_conv_paths(max_ell, hidden_l) == [tuple(p) for p in EQ.conv_paths(max_ell, hidden_l)]


@pytest.mark.parametrize("eq", [False, True], ids=["contractions0", "contractions0and1"])
@pytest.mark.parametrize("max_ell", [0, 1, 2, 3])
@pytest.mark.parametrize("corr", [1, 2, 3])
def test_term_builder_reproduces_u_contraction(shim, max_ell, corr, eq):
    if eq and max_ell == 0:
        pytest.skip("a 1o output needs max_ell >= 1")
    nsh, Cr, C, n = (max_ell + 1) ** 2, 32, 64, 23
    mods = M.make_contraction(max_ell, corr, Cr, eq, seed=7 + max_ell + 3 * corr)
    terms = M.build_terms(shim, mods, nsh)
    w, _ = M.stack_weights(mods, C)
    c = M.gen_graph(n, 5)
    z = c["type"][:n].long()
    A = M.rnd(c["g"], nsh, n, C, s=0.7, Cr=Cr)
    f = M.symc_fn(mods, c, n, C, nsh, eq)
    ref = M.multilinear(f, dict(A=A))
    got = M.symc_terms_fwd(terms, A, w, z, eq, nsh).reshape(-1)
    # the terms carry fp32 coefficients: a few roundings of each term at most
    assert KU.max_err(got, ref.x, ref.s) < 3 * 2.0 ** -24, KU.max_err(got, ref.x, ref.s)
    gB = M.rnd(c["g"], 4 if eq else 1, n, C, Cr=Cr)
    r = M.multilinear(f, dict(A=A), g=gB.reshape(-1), wrt=("A",))
    gA = M.symc_terms_bwd(terms, A, w, z, gB, nsh, eq)
    assert KU.max_err(gA, r["A"].x, r["A"].s) < 3 * 2.0 ** -24


# ------------------------------------------------------------------------------------------------ scales
def test_scales_bound_values():
    c = M.gen_graph(37, 9, empty=3, heavy=300)
    for zbl, agnesi in ((False, False), (True, True)):
        core = M.core_params(zbl, agnesi)
        for k, v in M.edge_geom_ref(c, 8, 16, core).items():
            assert bool((v.s >= v.x.abs() * (1 - 1e-12)).all()), k
        g = c["g"]
        N = c["N"]
        r = M.edge_final_ref(c, 8, 16, core, M.rnd(g, c["E"], 64), M.rnd(g, c["E"], 16), M.rnd(g, N, 3),
                             M.rnd(g, 9).double(), M.rnd(g, N, 12), 0.5 + torch.rand(N, generator=g))
        for k, v in r.items():
            assert bool((v.s >= v.x.abs() * (1 - 1e-12)).all()), k
    # the hand-written per-edge gradient (gd u + (h - pr u) / d) equals autograd's
    core = M.core_params(True, True)
    e = c["E"]
    g_eb, gY = M.rnd(c["g"], e, 64), M.rnd(c["g"], e, 16)
    v = M.d64(c["e_vec"][:, :3]).requires_grad_(True)
    wz = torch.full((e,), 1.3, dtype=torch.float64)
    with torch.enable_grad():
        (gv,) = torch.autograd.grad(M.edge_energy(v, c, 8, 16, core, g_eb, gY, wz).sum(), v)
    vd = v.detach()
    d = vd.norm(dim=1)
    u = vd / d[:, None]
    deb = torch.func.jvp(lambda x: M.radial_basis(x, c, 8, core), (d,), (torch.ones_like(d),))[1][:, :8]
    dV = torch.func.jvp(lambda x: M.zbl_edge(x, c, core), (d,), (torch.ones_like(d),))[1]
    gd = (M.d64(g_eb)[:, :8] * deb).sum(1) + 1.3 * dV
    gy = M.d64(gY).clone()
    gy[:, 0] = 0
    # h: gradient of sum gY Y(u) in the unit vector's components, tangential part only (sh_basis normalises)
    ht = torch.stack([(gy * dy).sum(1) for dy in M._jvp_cols(lambda x: M.sh(x, 16), vd, range(3))], 1)
    hand = gd[:, None] * u + ht
    assert torch.allclose(hand, gv, rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------------ mutants
def test_edge_geom_mutants():
    c = M.gen_graph(37, 8, empty=3, heavy=300)
    core = M.core_params(False, True)
    ref = M.edge_geom_ref(c, 8, 16, core)
    for mut in ("y_swap_11_13", "no_last_bessel"):
        m = M.edge_geom_ref(c, 8, 16, core, mut=(mut,))
        sharp(mut, "edge_geom", [(m[k].x, ref[k]) for k in ref])


def test_edge_final_mutants():
    c = M.gen_graph(37, 512, empty=3, heavy=300)
    g, E, N = c["g"], c["E"], c["N"]
    core = M.core_params(True, True)
    g_eb, gY = M.rnd(g, E, 64, s=0.5), M.rnd(g, E, 16, s=0.5)
    F0, v0, av0 = M.rnd(g, N, 3), M.rnd(g, 9).double(), M.rnd(g, N, 12)
    wv = 0.5 + torch.rand(N, generator=g)
    ref = M.edge_final_ref(c, 8, 16, core, g_eb, gY, F0, v0, av0, wv)
    for mut in ("y_swap_11_13", "no_last_bessel", "no_env_df", "no_agnesi_dx", "no_pr", "vir_transposed",
                "atom_vir_all_dst", "wgt_twice"):
        m = M.edge_final_ref(c, 8, 16, core, g_eb, gY, F0, v0, av0, wv, mut=(mut,))
        sharp(mut + " (edge_final)", "edge_final", [(m[k].x, ref[k]) for k in ref])


def test_msg_eq_mutants():
    Cr, C, max_ell = 32, 64, 3
    c = M.gen_graph(37, 43, empty=3, heavy=300)
    paths, _, _, _ = M.eq_layout(max_ell)
    g = torch.Generator().manual_seed(203)
    E = c["E"]
    R = M.rnd(g, E, len(paths), C, Cr=Cr).reshape(E, -1)
    Y = M.sh(M.d64(c["e_vec"][:, :3]), 16).float()
    u = M.rnd(g, c["n_loc"], 4, C, Cr=Cr).reshape(c["n_loc"], -1)
    ref = M.multilinear(M.msg_eq_fn(c, C, max_ell), dict(R=R, Y=Y, u=u))
    for mut in ("cg_sign_l3", "paths_swapped", "no_sqrt_2l1"):
        m = M.multilinear(M.msg_eq_fn(c, C, max_ell, mut=(mut,)), dict(R=R, Y=Y, u=u))
        sharp(mut, "msg_eq", [(m.x, ref)])


def test_symc_mutants(shim):
    Cr, C, max_ell, corr = 32, 64, 3, 3
    for eq in (False, True):
        c = M.gen_graph(37, 333 + eq)
        n, nsh = c["n_own"], 16
        mods = M.make_contraction(max_ell, corr, Cr, eq, 333 + eq)
        terms = M.build_terms(shim, mods, nsh)
        w, _ = M.stack_weights(mods, C)
        A = M.rnd(c["g"], nsh, n, C, s=0.7, Cr=Cr)
        gB = M.rnd(c["g"], 4 if eq else 1, n, C, Cr=Cr)
        f = M.symc_fn(mods, c, n, C, nsh, eq)
        ref = M.multilinear(f, dict(A=A))
        rb = M.multilinear(f, dict(A=A), g=gB.reshape(-1), wrt=("A",))["A"]
        muts = ["one_permutation", "drop_smallest_term", "kg_off_by_one", "elem_of_neighbour"]
        muts += ["o_slots_1_3_swapped"] if eq else []
        for mut in muts:
            m = M.multilinear(M.symc_fn(mods, c, n, C, nsh, eq, mut=(mut,)), dict(A=A))
            mb = M.multilinear(M.symc_fn(mods, c, n, C, nsh, eq, mut=(mut,)), dict(A=A), g=gB.reshape(-1),
                               wrt=("A",))["A"]
            sharp(f"{mut} (eq={eq})", "symc", [(m.x, ref), (mb.x, rb)])
        z = c["type"][:n].long()
        mb = M.symc_terms_bwd(terms, A, w, z, gB, nsh, eq, mut=("repeat_once",))
        sharp(f"repeat_once (eq={eq})", "symc_bwd", [(mb, rb)])


def test_elem_mix_mutants():
    Cr, C, L1, nsh = 32, 64, 4, 16
    c = M.gen_graph(37, 76)
    g, n = c["g"], c["n_own"]
    W = M.rnd(g, len(M.ELEMS), L1, C, C, s=C ** -0.5, Cr=Cr)
    W[..., Cr:, :] = 0.0
    x = M.rnd(g, nsh, n, C, Cr=Cr)
    ref = M.multilinear(M.elem_mix_fn(c, n, C, L1, nsh), dict(W=W, x=x))
    for mut in ("l1_block_on_l2", "elem_of_neighbour"):
        m = M.multilinear(M.elem_mix_fn(c, n, C, L1, nsh, mut=(mut,)), dict(W=W, x=x))
        sharp(mut + " (elem_mix)", "elem_mix", [(m.x, ref)])


def test_readout_mutants():
    Cr, C, H = 32, 64, 16
    c = M.gen_graph(37, 126)
    g, n, N = c["g"], c["n_own"], c["N"]
    pre = M.rnd(g, n, H, s=2.0)
    W1 = M.rnd(g, C, H, s=C ** -0.5)
    W1[Cr:] = 0.0
    w2 = M.rnd(g, H, s=1.6 * H ** -0.5)
    wv = 0.5 + torch.rand(N, generator=g)
    ref = M.readout_seed_ref(c, pre, W1, w2, 1.3, wv)
    for mut in ("silu_p_as_sigma", "wgt_twice"):
        sharp(mut + " (seed)", "readout", [(M.readout_seed_ref(c, pre, W1, w2, 1.3, wv, mut=(mut,)).x, ref)])
    h = M.rnd(g, n, C, Cr=Cr)
    el = M.rnd(g, n)
    E0 = torch.linspace(-3.0, -1.0, len(M.ELEMS), dtype=torch.float64)
    ref = M.readout_final_ref(c, h, W1, w2, el, E0, 1.3, -0.2, wv)
    for mut in ("e0_wrong_element", "wgt_twice"):
        m = M.readout_final_ref(c, h, W1, w2, el, E0, 1.3, -0.2, wv, mut=(mut,))
        sharp(mut + " (final)", "readout", [(m[k].x, ref[k]) for k in ("energy", "eps")])
