"""CPU checks of the 0e+1o+2e MACE oracle (tests/mace_l2_ref.py), of the coupling lists the engine compiles in for it
(csrc/mace_cg_l2.cuh), of the engine's host path list and term builder through the kernel shim, and of the
wrapper's recognition of such models."""
from __future__ import annotations

import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, si_diamond
from oracle.mace_ref import _random_rotation, l_of_index, wigner_d
from tests import kernel_units_ref as KU
from tests import mace_l2_units_ref as LU
from tests import mace_eq_ref as EQ
from tests import mace_units_ref as M
from tests.mace_eq_ref import make_mace_eq
from tests.mace_l2_ref import (RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock, atomic_virials_ref,
                               conv_paths, embed_medium, make_cg, make_mace_l2, make_u_out, potential_ref)
from tests.test_ptxas_spills import nvcc

SYMS = ("Si", "C", "O")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def small(pbc=(True, True, True), seed=0):
    a = si_diamond(1, seed=seed)  # 8 atoms
    rng = np.random.default_rng(seed)
    sy = [SYMS[k] for k in rng.integers(0, 3, len(a))]
    return SimpleAtoms(sy, a.get_positions(), np.array(a.get_cell()), pbc=pbc)


def model(**kw):
    kw.setdefault("C", 8)
    kw.setdefault("r_max", 4.0)
    kw.setdefault("scale", 8.0)
    kw.setdefault("max_ell", 2)
    return make_mace_l2(**kw)


def _blk(D, l):
    return D[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2]


# ------------------------------------------------------------------------------------------ paths, couplings, U
def test_conv_path_counts():
    for max_ell, npl in ((2, [3, 4, 4]), (3, [3, 5, 5, 4])):
        p = conv_paths(max_ell, 2)
        assert [sum(q[2] == l for q in p) for l in range(max_ell + 1)] == npl
        assert sum((2 * l + 1) * n for l, n in enumerate(npl)) == {2: 35, 3: 71}[max_ell]
        assert conv_paths(max_ell, 1) == [q for q in p if q[0] <= 1]  # the 0e+1o paths keep their relative order


@pytest.mark.parametrize("ls", sorted({p for p in conv_paths(3, 2) if p[0] == 2}))
def test_cg_of_2e_paths_equivariant(ls):
    cg = make_cg(*ls)
    assert abs(torch.linalg.norm(cg).item() - 1.0) < 1e-12
    rng = np.random.default_rng(78)
    for _ in range(2):
        D = wigner_d(_random_rotation(rng), 3, rng)
        T = torch.einsum("ai,bj,ck,ijk->abc", _blk(D, ls[0]), _blk(D, ls[1]), _blk(D, ls[2]), cg)
        assert (T - cg).abs().max() < 1e-12


def test_engine_cg_table_l2_equals_make_cg():
    """csrc/mace_cg_l2.cuh (compiled into k_mace_msg_l2 / _bwd) against make_cg and conv_paths"""
    text = open(os.path.join(ROOT, "distmlip_b200", "csrc", "mace_cg_l2.cuh")).read()
    for L in (2, 3):
        body = text.split(f"#define MACE_CG_L2_{L}(X)")[1].split("#define")[0]
        got = {(int(p), int(iu), int(iy), int(s)): float(v) for p, iu, iy, s, v in
               re.findall(r"X\((\d+), (\d+), (\d+), (\d+), ([-+0-9.e]+)f\)", body)}
        paths, per, base, _ = LU.l2_layout(L)
        want = {}
        for p, (li, ls, lo) in enumerate(paths):
            j = per[lo].index(p)
            cg = make_cg(li, ls, lo) * math.sqrt(2 * lo + 1)
            for m1, m2, m3 in itertools.product(range(2 * li + 1), range(2 * ls + 1), range(2 * lo + 1)):
                if abs(cg[m1, m2, m3]) > 1e-9:
                    want[(p, li * li + m1, ls * ls + m2, base[lo] + m3 * len(per[lo]) + j)] = cg[m1, m2, m3].item()
        assert got.keys() == want.keys(), L
        assert max(abs(got[k] - want[k]) for k in want) < 1e-8


@pytest.mark.parametrize("max_ell,nu", [(2, 1), (2, 2), (2, 3), (3, 1), (3, 2)])
def test_u_2e_symmetric_orthonormal_equivariant(max_ell, nu):
    U = make_u_out(max_ell, nu, 2)
    n, K = (max_ell + 1) ** 2, U.shape[-1]
    assert U.shape == (5,) + (n,) * nu + (K,) and K > 0
    flat = U.reshape(-1, K)
    assert torch.allclose(flat.T @ flat, torch.eye(K, dtype=torch.float64), atol=1e-12)
    for perm in itertools.permutations(range(1, nu + 1)):
        assert (U - U.permute(0, *perm, nu + 1)).abs().max() < 1e-12
    rng = np.random.default_rng(322)
    D = wigner_d(_random_rotation(rng), max_ell, rng)
    par = torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64))
    for Di, Do in ((D, _blk(D, 2)), (par, torch.eye(5, dtype=torch.float64))):  # 2e: even under inversion
        T = torch.movedim(torch.tensordot(U, Do, dims=([0], [1])), -1, 0)
        for ax in range(nu):
            T = torch.movedim(torch.tensordot(T, Di, dims=([1 + ax], [1])), -1, 1 + ax)
        assert (T - U).abs().max() < 1e-12


# ------------------------------------------------------------------------------------------ the model
def test_state_dict_names_and_shapes():
    C, ne = 8, 3
    sd = model(C=C, num_interactions=3, max_ell=3).state_dict()
    assert sd["interactions.1.linear_up.weight"].numel() == 3 * C * C
    assert sd["interactions.1.conv_tp_weights.layer3.weight"].shape[1] == 17 * C
    assert sd["interactions.1.linear.weight"].numel() == 17 * C * C
    assert sd["interactions.1.skip_tp.weight"].numel() == 3 * C * ne * C  # 0e->0e, 1o->1o, 2e->2e
    assert sd["interactions.2.skip_tp.weight"].numel() == C * ne * C
    assert sd["products.0.symmetric_contractions.contractions.2.U_matrix_2"].shape[0] == 5
    assert sd["products.1.linear.weight"].numel() == 3 * C * C
    assert sd["products.2.linear.weight"].numel() == C * C
    assert not any(k.startswith("products.2.symmetric_contractions.contractions.1") for k in sd)


def test_energy_invariances():
    m = model(seed=1, num_interactions=3)
    a = small(seed=1)
    E0 = potential_ref(m, a, calc_forces=False)[0].item()
    cell, pos = np.array(a.get_cell()), a.get_positions()
    R = _random_rotation(np.random.default_rng(5))
    for c, p in ((cell @ R.T, pos @ R.T), (-cell, -pos), (cell, pos + np.array([0.3, -1.1, 2.0]))):
        E = potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), p, c), calc_forces=False)[0].item()
        assert abs(E - E0) < 1e-10 * max(1.0, abs(E0))


def test_h1_2e_block_transforms_with_d2():
    m = model(seed=4, max_ell=3)
    a = small(seed=4)
    rng = np.random.default_rng(9)
    R = _random_rotation(rng)
    D = wigner_d(R, 3, rng)
    t0, t1 = {}, {}
    potential_ref(m, a, calc_forces=False, taps=t0)
    potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), a.get_positions() @ R.T, np.array(a.get_cell()) @ R.T),
                  calc_forces=False, taps=t1)
    h0, h1 = t0["h1"], t1["h1"]  # [n, 9, C]
    assert h0.shape == (len(a), 9, 8)
    tol = 1e-9 * max(1.0, h0.abs().max().item())
    assert (h1[:, 0] - h0[:, 0]).abs().max() < tol
    assert (h1[:, 1:4] - torch.einsum("ij,njc->nic", _blk(D, 1), h0[:, 1:4])).abs().max() < tol
    assert (h1[:, 4:9] - torch.einsum("ij,njc->nic", _blk(D, 2), h0[:, 4:9])).abs().max() < tol
    assert h0[:, 4:9].abs().max() > 1e-3


@pytest.mark.parametrize("pbc", [(True, True, True), (False, False, False)])
def test_forces_and_stress_finite_differences(pbc):
    cls = [RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock, RealAgnosticResidualInteractionBlock]
    m = model(seed=2, correlation=3, num_interactions=3, interaction_classes=cls)
    a = small(pbc=pbc, seed=2)
    if not any(pbc):
        a = SimpleAtoms(a.get_chemical_symbols(), a.get_positions(), np.eye(3) * 30.0, pbc=pbc)
    E, F, S, _ = potential_ref(m, a)
    h = 1e-5
    pos, cell = a.get_positions(), np.array(a.get_cell())
    en = lambda p, c: potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), p, c, pbc=pbc), calc_forces=False,  # noqa: E731
                                    calc_stresses=False)[0].item()
    for i, k in ((0, 0), (3, 2), (5, 1)):
        dp = np.zeros_like(pos)
        dp[i, k] = h
        fd = -(en(pos + dp, cell) - en(pos - dp, cell)) / (2 * h)
        assert abs(fd - F[i, k].item()) < 1e-6 * max(1.0, abs(fd))
    if all(pbc):
        for (i, j) in ((0, 0), (1, 2)):
            eps = np.zeros((3, 3))
            eps[i, j] = eps[j, i] = h / 2 if i != j else h
            fd = (en(pos @ (np.eye(3) + eps), cell @ (np.eye(3) + eps)) -
                  en(pos @ (np.eye(3) - eps), cell @ (np.eye(3) - eps))) / (2 * h)
            vol = abs(np.linalg.det(cell))
            assert abs(fd / vol * 160.21766208 - S[i, j].item()) < 1e-5 * max(1.0, abs(S[i, j].item()))


def test_atomic_energies_and_virials_sum_rules():
    m = model(seed=3)
    a = small(seed=3)
    E, _, S, eps = potential_ref(m, a)
    assert abs(eps.sum().item() - E.item()) < 1e-10 * max(1.0, abs(E.item()))
    w = atomic_virials_ref(m, a)
    vol = abs(np.linalg.det(np.array(a.get_cell())))
    assert (w.sum(0) - S * vol / 160.21766208).abs().max() < 1e-9 * max(1.0, w.abs().max().item())


@pytest.mark.parametrize("T,cls", [(2, None), (3, "residual"), (3, "plain")])
def test_zeroed_2e_reproduces_the_0e_1o_model(T, cls):
    kw = dict(C=8, max_ell=3, correlation=2, r_max=4.0, num_interactions=T)
    if cls is not None:
        names = ["RealAgnosticInteractionBlock"] + [("RealAgnosticResidualInteractionBlock" if cls == "residual" else
                                                     "RealAgnosticInteractionBlock")] * (T - 1)
        kw_l2 = dict(kw, interaction_classes=[globals()[n] for n in names])
        kw_eq = dict(kw, interaction_classes=[getattr(EQ, n) for n in names])
    else:
        kw_l2 = kw_eq = kw
    med = make_mace_eq(seed=20 + T, **kw_eq)
    large = embed_medium(make_mace_l2(seed=40 + T, **kw_l2), med)
    a = small(seed=T)
    E1, F1, S1, e1 = potential_ref(med, a)
    E2, F2, S2, e2 = potential_ref(large, a)
    assert abs(E1.item() - E2.item()) < 1e-10 * max(1.0, abs(E1.item()))
    assert (F1 - F2).abs().max() < 1e-10 and (S1 - S2).abs().max() < 1e-9 and (e1 - e2).abs().max() < 1e-10


# ------------------------------------------------------------------------------------------ wrapper
def _describe(m):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    return ScaleShiftMACE_Dist.from_existing(m)._describe()


@pytest.mark.parametrize("T", [2, 3])
@pytest.mark.parametrize("max_ell", [2, 3])
def test_wrapper_accepts_0e_1o_2e(T, max_ell):
    d = _describe(model(C=32, num_interactions=T, max_ell=max_ell, correlation=2))
    assert d.hidden_max_l == 2 and d.max_ell == max_ell and d.num_interactions == T and d.channels == 32
    assert list(d.hidden_mul) == [32, 32, 32, 0]
    assert list(_describe(make_mace_eq(C=32, r_max=4.0, max_ell=max_ell, num_interactions=T)).hidden_mul) == [32, 32, 0, 0]


def _reject(m, match, edit=None):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    if edit is not None:
        edit(d._state_dict)
    with pytest.raises(NotImplementedError, match=match):
        d._describe()


def _irreps(m, text):
    for it in m.interactions:
        it.hidden_irreps = text
    return m


def test_wrapper_refusals():
    l2 = lambda: model(C=32, max_ell=2, correlation=1)  # noqa: E731
    _reject(_irreps(l2(), "32x0e+32x1o+32x2e+32x3o"), "hidden l = 3")
    _reject(_irreps(l2(), "32x0e+32x1o+64x2e"), "unequal multiplicities")
    _reject(_irreps(l2(), "32x0e+32x1o+32x2o"), "only 1o and 2e")
    _reject(_irreps(make_mace_eq(C=32, r_max=4.0, max_ell=1, correlation=1), "32x0e+32x1o+32x2e"), "max_ell >= 2")
    pc = "products.0.symmetric_contractions.contractions."

    def bare():
        mm = l2()
        for it in mm.interactions:
            del it.hidden_irreps
        return mm

    _reject(bare(), "hidden l = 3", lambda sd: sd.__setitem__(pc + "3.U_matrix_1", torch.zeros(7, 9, 1)))
    _reject(bare(), r"hidden l > 1 \(2e\)", lambda sd: sd.__setitem__(pc + "2.U_matrix_1", torch.zeros(7, 9, 1)))
    _reject(bare(), "unequal multiplicities",
            lambda sd: sd.__setitem__(pc + "2.weights_max", torch.zeros(3, sd[pc + "2.weights_max"].shape[1], 64)))
    _reject(bare(), r"hidden l > 1 \(2e\)",
            lambda sd: sd.__setitem__("products.0.linear.weight", torch.zeros(2 * 32 * 32)))
    _reject(bare(), r"hidden l > 1 \(2e\)",
            lambda sd: sd.__setitem__("interactions.1.conv_tp_weights.layer3.weight", torch.zeros(64, 10 * 32)))


# ------------------------------------------------------------------------------------------ engine host code (shim)
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    if nvcc() is None:
        pytest.skip("nvcc not found")
    return KU.Shim(LU.build_shim_l2(tmp_path_factory.mktemp("kernel_shim_l2")))


def test_engine_conv_paths_hidden_l2(shim):
    for max_ell in (2, 3):
        assert shim.mace_conv_paths(max_ell, 2) == [tuple(p) for p in conv_paths(max_ell, 2)]


@pytest.mark.parametrize("max_ell,corr", [(2, 1), (2, 3), (3, 2), (3, 3)])
def test_term_builder_2e_reproduces_u_contraction(shim, max_ell, corr):
    nsh, Cr, C, n = (max_ell + 1) ** 2, 32, 64, 23
    mods = LU.make_contraction_l2(max_ell, corr, Cr, seed=9 + max_ell + 3 * corr)
    terms = LU.build_terms_l2(shim, mods, nsh)
    w, _ = M.stack_weights(mods, C)
    c = M.gen_graph(n, 5)
    z = c["type"][:n].long()
    A = M.rnd(c["g"], nsh, n, C, s=0.7, Cr=Cr)
    ref = M.multilinear(LU.symc_l2_fn(mods, c, n, C, nsh), dict(A=A))
    got = LU.terms_fwd9(terms, A, w, z).reshape(-1)
    assert KU.max_err(got, ref.x, ref.s) < 3 * 2.0 ** -24, KU.max_err(got, ref.x, ref.s)
    slots = {(int(t) & 0xFFFFFFFF) >> 28 for t in terms[:, 0]}
    assert slots == set(range(9))  # slot 8 sets bit 31 of the packed index
