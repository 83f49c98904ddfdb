"""CPU checks of the MACE oracle (oracle/mace_ref.py) and of the MACE wrapper's configuration checks."""
from __future__ import annotations

import itertools

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, si_diamond
from oracle.mace_ref import (_random_rotation, l_of_index, make_mace, make_u, potential_ref, sh_basis, wigner_d)

SYMS = ("Si", "C", "O")


def small(pbc=(True, True, True), seed=0):
    a = si_diamond(1, seed=seed)  # 8 atoms, 5.43 A cell
    rng = np.random.default_rng(seed)
    sy = [SYMS[k] for k in rng.integers(0, 3, len(a))]
    return SimpleAtoms(sy, a.get_positions(), np.array(a.get_cell()), pbc=pbc)


def model(**kw):
    kw.setdefault("C", 32)
    kw.setdefault("r_max", 4.0)
    kw.setdefault("scale", 8.0)
    return make_mace(**kw)


@pytest.mark.parametrize("max_ell", [1, 2, 3])
@pytest.mark.parametrize("nu", [1, 2, 3])
def test_u_symmetric_invariant_orthonormal(max_ell, nu):
    U = make_u(max_ell, nu)
    K = U.shape[-1]
    flat = U.reshape(-1, K)
    assert torch.allclose(flat.T @ flat, torch.eye(K, dtype=torch.float64), atol=1e-12)
    for perm in itertools.permutations(range(nu)):
        assert (U - U.permute(*perm, nu)).abs().max() < 1e-12
    rng = np.random.default_rng(123)
    gens = [wigner_d(_random_rotation(rng), max_ell, rng),
            torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64))]
    for D in gens:
        T = U
        for ax in range(nu):
            T = torch.movedim(torch.tensordot(T, D, dims=([ax], [1])), -1, ax)
        assert (T - U).abs().max() < 1e-12


def test_sh_component_normalisation():
    Y = sh_basis(torch.randn(50, 3, dtype=torch.float64), 3)
    for l in range(4):
        assert torch.allclose((Y[:, l * l:(l + 1) ** 2] ** 2).sum(1), torch.full((50,), 2.0 * l + 1, dtype=torch.float64))


def test_energy_invariances():
    m = model(seed=1)
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


@pytest.mark.parametrize("pbc", [(True, True, True), (True, True, False), (False, False, False)])
def test_forces_and_stress_finite_differences(pbc):
    m = model(seed=2, correlation=3)
    a = small(pbc=pbc, seed=2)
    if not any(pbc):
        a = SimpleAtoms(a.get_chemical_symbols(), a.get_positions(), np.eye(3) * 30.0, pbc=pbc)
    E, F, S, _ = potential_ref(m, a)
    h = 1e-5
    pos, cell = a.get_positions(), np.array(a.get_cell())
    en = lambda p, c: potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), p, c, pbc=pbc), calc_forces=False,
                                    calc_stresses=False)[0].item()
    for i, k in ((0, 0), (3, 2), (5, 1)):
        dp = np.zeros_like(pos)
        dp[i, k] = h
        fd = -(en(pos + dp, cell) - en(pos - dp, cell)) / (2 * h)
        assert abs(fd - F[i, k].item()) < 1e-6
    if all(pbc):
        for (i, j) in ((0, 0), (1, 2)):
            eps = np.zeros((3, 3))
            eps[i, j] = eps[j, i] = h / 2 if i != j else h
            fd = (en(pos @ (np.eye(3) + eps), cell @ (np.eye(3) + eps)) -
                  en(pos @ (np.eye(3) - eps), cell @ (np.eye(3) - eps))) / (2 * h)
            vol = abs(np.linalg.det(cell))
            assert abs(fd / vol * 160.21766208 - S[i, j].item()) < 1e-5


def test_atomic_energies_sum():
    m = model(seed=3)
    E, _, _, eps = potential_ref(m, small(seed=3))
    assert abs(eps.sum().item() - E.item()) < 1e-10


def _reject(m, match):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    with pytest.raises(NotImplementedError, match=match):
        d._describe()


def test_wrapper_rejects_unsupported_options():
    _reject(model(C=48), "multiple of 32")
    _reject(model(C=160), "multiple of 32")
    m = model()
    m.heads = ["a", "b"]
    _reject(m, "multi-head")
    m = model()
    m.pair_repulsion = True
    _reject(m, "pair_repulsion")
    m = model()
    m.radial_embedding.distance_transform = torch.nn.Identity()
    _reject(m, "distance_transform")
    m = model()
    m.interactions[0].__class__ = type("RealAgnosticDensityInteractionBlock", (type(m.interactions[0]),), {})
    _reject(m, "RealAgnosticDensityInteractionBlock")
    m = model(radial_mlp=(128,))
    _reject(m, "at most 64")
    m = model()
    m.readouts[0].__class__ = type("NonLinearReadoutBlock", (type(m.readouts[0]),), {})
    _reject(m, "readouts.0")


def _reject_sd(edit, match):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(model())
    edit(d._state_dict)
    with pytest.raises(NotImplementedError, match=match):
        d._describe()


PC = "products.0.symmetric_contractions.contractions."


def test_wrapper_rejects_unsupported_state_dicts():
    _reject_sd(lambda sd: sd.__setitem__(PC + "0.U_matrix_4", torch.zeros(1)), "correlation=4")
    _reject_sd(lambda sd: sd.__setitem__(PC + "0.U_matrix_1", torch.zeros(25, 1)), "max_ell <= 3")
    _reject_sd(lambda sd: sd.__setitem__(PC + "0.U_matrix_1", torch.zeros(3, 16, 1)), "equivariant hidden")
    _reject_sd(lambda sd: sd.__setitem__(PC + "1.weights_max", torch.zeros(1)), "equivariant hidden")
    _reject_sd(lambda sd: sd.__setitem__("atomic_dipoles_fn.weight", torch.zeros(1)), "dipole")
    _reject_sd(lambda sd: sd.__setitem__("radial_embedding.gaussian_fn.centers", torch.zeros(8)), "Bessel")
    _reject_sd(lambda sd: sd.pop("radial_embedding.bessel_fn.bessel_weights"), "Bessel")
    _reject_sd(lambda sd: sd.__setitem__("pair_repulsion_fn.a", torch.zeros(1)), "pair_repulsion")


def test_wrapper_rejects_non_mace():
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    with pytest.raises(TypeError, match="ScaleShiftMACE"):
        ScaleShiftMACE_Dist.from_existing(torch.nn.Linear(2, 2))
