"""CPU checks of the MACE oracle with hidden features C x 0e + C x 1o (tests/mace_eq_ref.py), of the coupling
table the engine compiles in (csrc/mace_cg.cuh), and of the wrapper's recognition of such models."""
from __future__ import annotations

import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, si_diamond
from oracle.mace_ref import _random_rotation, l_of_index, make_mace, species_index, wigner_d
from tests.mace_eq_ref import (RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock, conv_paths, make_cg,
                               make_mace_eq, make_u_vec, potential_ref)
from oracle.graph_ref import neighbor_list

SYMS = ("Si", "C", "O")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def small(pbc=(True, True, True), seed=0):
    a = si_diamond(1, seed=seed)  # 8 atoms, 5.43 A cell
    rng = np.random.default_rng(seed)
    sy = [SYMS[k] for k in rng.integers(0, 3, len(a))]
    return SimpleAtoms(sy, a.get_positions(), np.array(a.get_cell()), pbc=pbc)


def model(**kw):
    kw.setdefault("C", 32)
    kw.setdefault("r_max", 4.0)
    kw.setdefault("scale", 8.0)
    return make_mace_eq(**kw) if kw.pop("max_L", 1) else make_mace(**kw)


def _d(rng, lmax=3):
    return wigner_d(_random_rotation(rng), lmax, rng)


def _blk(D, l):
    return D[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2]


def test_conv_paths_order():
    assert conv_paths(3, 1) == [(0, 0, 0), (1, 1, 0), (0, 1, 1), (1, 0, 1), (1, 2, 1), (0, 2, 2), (1, 1, 2), (1, 3, 2),
                                (0, 3, 3), (1, 2, 3)]
    assert [len(conv_paths(L, 1)) for L in (1, 2, 3)] == [4, 7, 10]
    assert conv_paths(2, 0) == [(0, 0, 0), (0, 1, 1), (0, 2, 2)]


@pytest.mark.parametrize("ls", [p for p in sorted(set(conv_paths(3, 1)))])
def test_cg_equivariant_normalised_signed(ls):
    cg = make_cg(*ls)
    assert abs(torch.linalg.norm(cg).item() - 1.0) < 1e-12
    first = cg.reshape(-1)[cg.reshape(-1).abs() > 1e-6][0]
    assert first > 0  # the sign rule
    rng = np.random.default_rng(77)
    for _ in range(2):
        D = _d(rng)
        T = torch.einsum("ai,bj,ck,ijk->abc", _blk(D, ls[0]), _blk(D, ls[1]), _blk(D, ls[2]), cg)
        assert (T - cg).abs().max() < 1e-12
    if ls[0] == 0:  # (0, l) -> l: sqrt(2l + 1) CG is the identity (the path constant 1 of the scalar layers)
        eye = torch.eye(2 * ls[1] + 1, dtype=torch.float64)
        assert (cg[0] * math.sqrt(2 * ls[2] + 1) - eye).abs().max() < 1e-12


def test_engine_cg_table_equals_make_cg():
    """csrc/mace_cg.cuh (compiled into k_mace_msg_eq / _bwd) against make_cg and conv_paths"""
    text = open(os.path.join(ROOT, "distmlip_b200", "csrc", "mace_cg.cuh")).read()
    for L in (1, 2, 3):
        body = text.split(f"#define MACE_CG_{L}(X)")[1].split("#define")[0]
        got = {(int(p), int(iu), int(iy), int(s)): float(v) for p, iu, iy, s, v in
               re.findall(r"X\((\d+), (\d+), (\d+), (\d+), ([-+0-9.e]+)f\)", body)}
        paths = conv_paths(L, 1)
        npl = [sum(1 for p in paths if p[2] == l) for l in range(L + 1)]
        base = [sum((2 * k + 1) * npl[k] for k in range(l)) for l in range(L + 1)]
        want, seen = {}, [0] * (L + 1)
        for p, (li, ls, lo) in enumerate(paths):
            j, seen[lo] = seen[lo], seen[lo] + 1
            cg = make_cg(li, ls, lo) * math.sqrt(2 * lo + 1)
            for m1, m2, m3 in itertools.product(range(2 * li + 1), range(2 * ls + 1), range(2 * lo + 1)):
                if abs(cg[m1, m2, m3]) > 1e-9:
                    want[(p, li * li + m1, ls * ls + m2, base[lo] + m3 * npl[lo] + j)] = cg[m1, m2, m3].item()
        assert got.keys() == want.keys(), L
        assert max(abs(got[k] - want[k]) for k in want) < 1e-8


@pytest.mark.parametrize("max_ell", [1, 2, 3])
@pytest.mark.parametrize("nu", [1, 2, 3])
def test_u_vector_symmetric_orthonormal_equivariant(max_ell, nu):
    U = make_u_vec(max_ell, nu)
    n = (max_ell + 1) ** 2
    K = U.shape[-1]
    assert U.shape == (3,) + (n,) * nu + (K,) and K > 0
    flat = U.reshape(-1, K)
    assert torch.allclose(flat.T @ flat, torch.eye(K, dtype=torch.float64), atol=1e-12)
    for perm in itertools.permutations(range(1, nu + 1)):
        assert (U - U.permute(0, *perm, nu + 1)).abs().max() < 1e-12
    rng = np.random.default_rng(321)
    D = wigner_d(_random_rotation(rng), max_ell, rng)
    par = torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64))
    for Di, Do in ((D, D[1:4, 1:4]), (par, -torch.eye(3, dtype=torch.float64))):
        T = torch.movedim(torch.tensordot(U, Do, dims=([0], [1])), -1, 0)
        for ax in range(nu):
            T = torch.movedim(torch.tensordot(T, Di, dims=([1 + ax], [1])), -1, 1 + ax)
        assert (T - U).abs().max() < 1e-12
    # one l-tuple of the input indices per basis tensor (U stays sparse)
    lidx = l_of_index(max_ell)
    for k in range(K):
        nz = U[..., k].nonzero()
        assert len({tuple(sorted(lidx[i] for i in row[1:].tolist())) for row in nz}) == 1


def test_layer0_is_the_scalar_interaction():
    """layer 0 takes 0e: the medium model's interactions.0 is the scalar model's block (same names and shapes)"""
    eq, sc = make_mace_eq(seed=5, C=32).state_dict(), make_mace(seed=5, C=32).state_dict()
    k0 = [k for k in sc if k.startswith("interactions.0.")]
    assert k0 and all(k in eq and eq[k].shape == sc[k].shape for k in k0)


def test_state_dict_names_and_shapes():
    C, ne = 32, 3
    sd = model(C=C, num_interactions=3, max_ell=3).state_dict()
    assert sd["interactions.0.linear_up.weight"].numel() == C * C
    assert sd["interactions.1.linear_up.weight"].numel() == 2 * C * C
    assert sd["interactions.1.conv_tp_weights.layer3.weight"].shape[1] == 10 * C
    assert sd["interactions.1.linear.weight"].numel() == 10 * C * C
    assert sd["interactions.1.skip_tp.weight"].numel() == 2 * C * ne * C  # 0e->0e, 1o->1o
    assert sd["interactions.2.skip_tp.weight"].numel() == C * ne * C  # last layer: 0e only
    assert sd["products.0.symmetric_contractions.contractions.1.U_matrix_2"].shape[0] == 3
    assert sd["products.1.linear.weight"].numel() == 2 * C * C
    assert sd["products.2.linear.weight"].numel() == C * C
    assert not any(k.startswith("products.2.symmetric_contractions.contractions.1") for k in sd)


def _rotated(a, R):
    return SimpleAtoms(a.get_chemical_symbols(), a.get_positions() @ R.T, np.array(a.get_cell()) @ R.T, pbc=a.get_pbc())


def test_energy_invariances():
    m = model(seed=1, num_interactions=3)
    a = small(seed=1)
    E0 = potential_ref(m, a, calc_forces=False)[0].item()
    cell, pos = np.array(a.get_cell()), a.get_positions()
    R = _random_rotation(np.random.default_rng(5))
    for c, p in ((cell @ R.T, pos @ R.T), (-cell, -pos), (cell, pos + np.array([0.3, -1.1, 2.0]))):
        E = potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), p, c), calc_forces=False)[0].item()
        assert abs(E - E0) < 1e-10 * max(1.0, abs(E0))
    perm = np.random.default_rng(2).permutation(len(a))
    sy = [a.get_chemical_symbols()[i] for i in perm]
    E = potential_ref(m, SimpleAtoms(sy, pos[perm], cell), calc_forces=False)[0].item()
    assert abs(E - E0) < 1e-10 * max(1.0, abs(E0))


def test_h1_vector_part_rotates():
    m = model(seed=4)
    a = small(seed=4)
    R = _random_rotation(np.random.default_rng(9))
    t0, t1 = {}, {}
    potential_ref(m, a, calc_forces=False, taps=t0)
    potential_ref(m, _rotated(a, R), calc_forces=False, taps=t1)
    h0, h1 = t0["h1"], t1["h1"]  # [n, 4, C]
    assert h0.shape == (len(a), 4, 32)
    assert (h1[:, 0] - h0[:, 0]).abs().max() < 1e-10
    # sh_basis l = 1 is sqrt(3) (x, y, z): D_1(g) = g
    rot = torch.einsum("ij,njc->nic", torch.as_tensor(R), h0[:, 1:])
    assert (h1[:, 1:] - rot).abs().max() < 1e-10 * max(1.0, h0.abs().max().item())
    assert h0[:, 1:].abs().max() > 1e-3


@pytest.mark.parametrize("pbc", [(True, True, True), (True, True, False), (False, False, False)])
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


def test_atomic_energies_sum():
    m = model(seed=3)
    E, _, _, eps = potential_ref(m, small(seed=3))
    assert abs(eps.sum().item() - E.item()) < 1e-10 * max(1.0, abs(E.item()))


# ------------------------------------------------------------------------------------------ wrapper
def _describe(m):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    return ScaleShiftMACE_Dist.from_existing(m)._describe()


@pytest.mark.parametrize("T", [2, 3])
@pytest.mark.parametrize("max_ell", [1, 2, 3])
def test_wrapper_accepts_0e_1o(T, max_ell):
    d = _describe(model(num_interactions=T, max_ell=max_ell))
    assert d.hidden_max_l == 1 and d.max_ell == max_ell and d.num_interactions == T and d.channels == 32
    assert _describe(model(num_interactions=T, max_ell=max_ell, max_L=0)).hidden_max_l == 0


def _reject(m, match, edit=None):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    if edit is not None:
        edit(d._state_dict)
    with pytest.raises(NotImplementedError, match=match):
        d._describe()


def test_wrapper_rejects_other_hidden_irreps():
    m = model()
    for it in m.interactions:
        it.hidden_irreps = "32x0e+32x1o+32x2e"
    _reject(m, "l > 1")
    m = model()
    for it in m.interactions:
        it.hidden_irreps = "32x0e+64x1o"
    _reject(m, "unequal multiplicities")
    m = model()
    for it in m.interactions:
        it.hidden_irreps = "32x0e+32x1e"
    _reject(m, "1e")
    # the same options seen in the state_dict alone (no hidden_irreps attribute)
    pc = "products.0.symmetric_contractions.contractions."

    def bare(**kw):
        mm = model(**kw)
        for it in mm.interactions:
            del it.hidden_irreps
        return mm

    _reject(bare(), "l > 1", lambda sd: sd.__setitem__(pc + "2.U_matrix_1", torch.zeros(5, 16, 1)))
    _reject(bare(), "unequal multiplicities",
            lambda sd: sd.__setitem__("interactions.1.linear_up.weight", torch.zeros(32 * 32 + 64 * 64)))
    _reject(bare(), "unequal multiplicities",
            lambda sd: sd.__setitem__(pc + "1.weights_max", torch.zeros(3, sd[pc + "1.weights_max"].shape[1], 64)))
    # a 1e hidden block changes conv_tp's paths: (1e, 1) -> 1o, (1e, 2) -> 2e, (1e, 3) -> 3o
    _reject(bare(), "only 1o",
            lambda sd: sd.__setitem__("interactions.1.conv_tp_weights.layer3.weight", torch.zeros(64, 7 * 32)))
    _reject(bare(), "equivariant hidden", lambda sd: sd.pop(pc + "1.U_matrix_1"))


def test_oracle_taps_and_species():
    m = model(seed=6)
    a = small(seed=6)
    taps = {}
    potential_ref(m, a, calc_forces=False, taps=taps)
    assert taps["h1"].shape == (8, 4, 32) and taps["h2"].shape == (8, 32) and taps["A1"].shape == (8, 16, 32)
    lat = np.array(a.get_cell())
    i1, i2, off, _, _ = neighbor_list(a.get_positions(), lat, np.ones(3, dtype=np.int64), 4.0, 0.0)
    assert len(i1) > 0 and species_index(m, a).shape == (8,)
