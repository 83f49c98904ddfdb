"""The tolerances of the 0e+1o+2e kernel-unit tests (tests/test_gpu_mace_l2_units.py) are sharp: on inputs built as
the GPU tests build them, what a subtly wrong kernel or term builder would compute (a float64 mutant) exceeds its
tolerance by at least MUTANT_MARGIN on some element."""
import pytest
import torch

from tests import kernel_units_ref as KU
from tests import mace_l2_units_ref as L
from tests import mace_units_ref as M

def sharp(name, tol, pairs):
    r = max(KU.max_err(mut, ref.x, ref.s) for mut, ref in pairs) / L.TOL[tol]
    print(f"mace l2 mutant {name:<24s} {r:.3g} x tol")
    assert r >= KU.MUTANT_MARGIN, (name, r)


@pytest.mark.parametrize("max_ell", [2, 3])
def test_msg_l2_mutants(max_ell):
    C, Cr = 64, 32
    c = M.gen_graph(37, 50 + max_ell, empty=3, heavy=300)
    paths, _, _, _ = L.l2_layout(max_ell)
    g = torch.Generator().manual_seed(7)
    E, nl = c["E"], c["n_loc"]
    R = M.rnd(g, E, len(paths), C, Cr=Cr).reshape(E, -1)
    Y = M.sh(M.d64(c["e_vec"][:, :3]), 16).float()
    u = M.rnd(g, nl, 9, C, Cr=Cr).reshape(nl, 9 * C)
    ref = M.multilinear(L.msg_l2_fn(c, C, max_ell), dict(R=R, Y=Y, u=u))
    for mut in ("cg_sign_2e", "drop_path_2"):
        m = M.multilinear(L.msg_l2_fn(c, C, max_ell, mut=(mut,)), dict(R=R, Y=Y, u=u))
        sharp(f"{mut} (max_ell {max_ell})", "msg_l2", [(m.x, ref)])


def test_elem_mix_rows9_mutants():
    C, Cr = 64, 32
    c = M.gen_graph(37, 81)
    g, n = c["g"], c["n_own"]
    W = M.rnd(g, len(M.ELEMS), 3, C, C, s=C ** -0.5, Cr=Cr)
    W[..., Cr:, :] = 0.0
    x = M.rnd(g, n, 9 * C)
    ref = M.multilinear(L.elem_mix_rows9_fn(c, n, C, 9 * C), dict(W=W, x=x))
    for mut in ("l1_mix_on_2e", "no_2e_skip"):
        m = M.multilinear(L.elem_mix_rows9_fn(c, n, C, 9 * C, mut=(mut,)), dict(W=W, x=x))
        sharp(mut, "elem_mix", [(m.x, ref)])


def test_symc_l2_slot_swap_mutant():
    max_ell, corr, Cr, C = 2, 2, 32, 64
    c = M.gen_graph(37, 612)
    g, n, nsh = c["g"], c["n_own"], (max_ell + 1) ** 2
    mods = L.make_contraction_l2(max_ell, corr, Cr, 612)
    A = M.rnd(g, nsh, n, C, s=0.7, Cr=Cr)
    ref = M.multilinear(L.symc_l2_fn(mods, c, n, C, nsh), dict(A=A))
    m = M.multilinear(L.symc_l2_fn(mods, c, n, C, nsh, mut=("slots_4_5_swapped",)), dict(A=A))
    sharp("slots_4_5_swapped", "symc", [(m.x, ref)])
