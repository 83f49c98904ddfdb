"""GPU: the heat flux of CHGNet and TensorNet (b2m_set_heat_flux / b2m_compute_heat_flux, DESIGN.md §10) against the
float64 unfolded-cell oracle (oracle/heat_flux_ref.py); the unfolded (masked) evaluation against a plain periodic
handle; partition independence in single-process groups; the off -> on -> off round trip; Potential_Dist,
PESCalculator_Dist and a few NVE steps; and, beyond the oracle's reach, invariance under a permutation of the atoms and
additivity under a repeat of the cell.

J_pot is compared relative to the size of its terms (oracle `scale`: max over components of sum_j |G_j . v_j| +
|(r_j - c)_a F~_j . v_j|), J_conv absolutely per unit of sum_i |v_i|.  tests/test_heat_flux_oracle.py checks that these
tolerances stay at least 10x below the error of plausible bugs."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
try:
    import ase  # noqa: F401
except ImportError:
    sys.path.insert(0, os.path.join(HERE, "stubs"))
    import ase  # noqa: F401

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.heat_flux_ref import heat_flux_ref, reach_of
from tests.test_gpu_atomic import (BIG, SCALING, TOL_EPS, TOL_W, engine_of, mixed, model_of, refs, set_structure)

pytestmark = pytest.mark.gpu
B2M_ERR_STATE = -6
TOL_J_REL = 1e-5   # |J_pot - J_pot_ref| / scale
TOL_JCONV = 2e-6   # eV, |J_conv - J_conv_ref| / sum_i |v_i|
# forces of the unfolded evaluation against a periodic handle: the fp32 atomics of two different graphs, then the fold
# (observed on an H100: 6.3e-8 eV/A for TensorNet; two plain evaluations already differ by 3e-8)
FTOL_ABS = 1.5e-7


def ftol(f0):
    return max(1e-8 * float(np.abs(f0).max()), FTOL_ABS)


def velocities(n, seed=0):
    return np.random.default_rng(seed).normal(scale=0.05, size=(n, 3))


def flux_oracle(family, atoms, v, **kw):
    model = model_of(family)
    return heat_flux_ref(model, atoms, v, element_refs=refs(model), dtype=torch.float64, **kw, **SCALING)


def check_flux(j_pot, j_conv, ref, v, what=""):
    dp = np.abs(j_pot - ref["j_pot"]).max() / ref["scale"]
    dc = np.abs(j_conv - ref["j_conv"]).max() / np.abs(v).sum()
    print(f"heat flux {what}: |dJ_pot| / scale {dp:.2e} (scale {ref['scale']:.3e}), |dJ_conv| / sum|v| {dc:.2e} eV")
    assert dp <= TOL_J_REL, dp
    assert dc <= TOL_JCONV, dc


def unfolded_engine(family, model, atoms, device=0, reach=None):
    eng = engine_of(family, model, device=device)
    eng.set_heat_flux(reach_of(model) if reach is None else reach)
    set_structure(eng, model, atoms)
    return eng


STRUCTURES = {
    "diamond64": lambda: mixed(si_diamond(2, sigma=0.15, seed=1)),
    "rough": lambda: mixed(rough_cell(300, seed=4), other="Ge", every=2),
}


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("structure", list(STRUCTURES))
def test_flux_matches_the_oracle(family, structure):
    atoms = STRUCTURES[structure]()
    model = model_of(family)
    v = velocities(len(atoms), 1)
    eng = unfolded_engine(family, model, atoms)
    e, f, s, (j_pot, j_conv) = eng.compute_heat_flux(v)
    ref = flux_oracle(family, atoms, v)
    c = eng.counts()
    print(f"{family} {structure}: {len(atoms)} atoms -> {c['n_own']} unfolded, {c['n_edges']} edges "
          f"(oracle {ref['n_unfolded']}, {ref['n_edges']})")
    assert c["n_own"] == ref["n_unfolded"] and c["n_edges"] == ref["n_edges"]
    check_flux(j_pot, j_conv, ref, v, f"{family} {structure}")
    assert abs(e - ref["energy"]) <= 1e-6 * abs(ref["energy"]) + 1e-6
    assert np.abs(f - ref["forces"]).max() <= 1e-5 * np.abs(ref["forces"]).max() + 1e-6
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_flux_matches_the_oracle_where_tiles_loop(family):
    """the unfolded graph has more than twice as many 128-edge tiles as resident CTAs (2 x 132), so the persistent
    kernels loop: TensorNet on a 4x4x2 diamond cell, CHGNet on 2x2x2 (its reach is 20 A)"""
    atoms = mixed(si_diamond(4, sigma=0.15, seed=9, nz=2) if family == "tensornet" else si_diamond(2, sigma=0.15, seed=9))
    model = model_of(family)
    v = velocities(len(atoms), 2)
    eng = unfolded_engine(family, model, atoms)
    _e, _f, _s, (j_pot, j_conv) = eng.compute_heat_flux(v)
    c = eng.counts()
    print(f"{family}: {c['n_own']} unfolded atoms, {c['n_edges']} edges, {c['n_edges'] // 128} edge tiles")
    assert c["n_edges"] // 128 > 2 * 132
    check_flux(j_pot, j_conv, flux_oracle(family, atoms, v), v, f"{family} tiles loop")
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_unfolded_evaluation_equals_the_periodic_one(family):
    atoms = mixed(si_diamond(2, sigma=0.15, seed=3))
    model = model_of(family)
    plain = engine_of(family, model)
    set_structure(plain, model, atoms)
    plain.set_atomic(True)
    e0, f0, s0 = plain.compute()
    eps0, w0 = plain.atomic()
    eng = unfolded_engine(family, model, atoms)
    eng.set_atomic(True)
    e1, f1, s1 = eng.compute()
    eps1, w1 = eng.atomic()
    df, ds = np.abs(f1 - f0).max(), np.abs(s1 - s0).max()
    print(f"unfolded vs periodic {family}: |dE| {abs(e1 - e0):.2e} eV, |dF| {df:.2e} eV/A, |dS| {ds:.2e} GPa, "
          f"|d eps| {np.abs(eps1 - eps0).max():.2e} eV, |dw| / max|w| {np.abs(w1 - w0).max() / np.abs(w0).max():.2e}")
    assert abs(e1 - e0) <= 1e-8 * abs(e0) + 1e-7
    assert df <= ftol(f0), df
    assert ds <= 1e-5 * np.abs(s0).max() + 1e-6, ds
    assert np.abs(eps1 - eps0).max() <= TOL_EPS
    assert np.abs(w1 - w0).max() <= TOL_W[family] * np.abs(w0).max()
    # the heat-flux call leaves the same periodic results behind
    e2, f2, s2, _j = eng.compute_heat_flux(velocities(len(atoms)))
    assert abs(e2 - e0) <= 1e-8 * abs(e0) + 1e-7 and np.abs(f2 - f0).max() <= ftol(f0)
    eps2, _w2 = eng.atomic()
    assert np.abs(eps2 - eps0).max() <= TOL_EPS
    plain.close()
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_partitions_of_a_group_give_the_same_flux(family):
    atoms = mixed(si_diamond(2, sigma=0.15, seed=5, nz=12))
    model = model_of(family)
    v = velocities(len(atoms), 3)
    ref = flux_oracle(family, atoms, v)
    for devs in ([0], [0, 0], [0, 0, 0]):
        eng = unfolded_engine(family, model, atoms, device=devs)
        _e, f, _s, (j_pot, j_conv) = eng.compute_heat_flux(v)
        assert eng.counts()["world"] == len(devs)
        check_flux(j_pot, j_conv, ref, v, f"{family} slab, {len(devs)} partitions")
        assert np.abs(f - ref["forces"]).max() <= 1e-5 * np.abs(ref["forces"]).max() + 1e-6
        eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_off_on_off_on_one_handle(family):
    from distmlip_b200._lib import B2MError

    atoms = mixed(si_diamond(2, sigma=0.15, seed=6))
    model = model_of(family)
    eng = engine_of(family, model)
    set_structure(eng, model, atoms)
    e0, f0, s0 = eng.compute()
    launches_off = eng.counts()["launches"]
    with pytest.raises(B2MError) as ei:
        eng.compute_heat_flux(velocities(len(atoms)))
    assert ei.value.code == B2M_ERR_STATE
    eng.set_heat_flux(reach_of(model))
    with pytest.raises(B2MError) as ei:  # the resident structure was built before the reach was set
        eng.compute_heat_flux(velocities(len(atoms)))
    assert ei.value.code == B2M_ERR_STATE
    set_structure(eng, model, atoms)
    e1, f1, s1, _j = eng.compute_heat_flux(velocities(len(atoms)))
    eng.set_heat_flux(0)
    set_structure(eng, model, atoms)
    e2, f2, s2 = eng.compute()
    assert eng.counts()["launches"] == launches_off
    assert eng.counts()["n_own"] == len(atoms)
    for e, f, s in ((e1, f1, s1), (e2, f2, s2)):
        assert abs(e - e0) <= 1e-8 * abs(e0) + 1e-7
        assert np.abs(f - f0).max() <= ftol(f0), (np.abs(f - f0).max(), ftol(f0))
        assert np.abs(s - s0).max() <= 1e-5 * np.abs(s0).max() + 1e-6
    eng.close()


@pytest.mark.parametrize("family,devices", [("chgnet", [0]), ("tensornet", [0, 0])])
def test_calculator_and_md(family, devices):
    from ase import Atoms

    from distmlip_b200.implementations.matgl import (CHGNet_Dist, MolecularDynamics, PESCalculator_Dist,
                                                     Potential_Dist, TensorNet_Dist)

    # 43 A along z: two periodic slabs wider than 2 (r_cut + r_bond); silicon only, as the ASE stand-in reports Z = 14
    base = si_diamond(2, sigma=0.15, seed=8, nz=8)
    atoms = Atoms(symbols=base.get_chemical_symbols(), positions=base.get_positions(), cell=base.get_cell(), pbc=True)
    v = velocities(len(atoms), 4)
    atoms.set_momenta(v * atoms.get_masses()[:, None])
    model = model_of(family)
    dm = (CHGNet_Dist if family == "chgnet" else TensorNet_Dist).from_existing(model)
    dm.enable_distributed_mode(devices)
    assert dm.heat_flux_reach() == reach_of(model)
    pot = Potential_Dist(model=dm, element_refs=refs(model), calc_heat_flux=True, **SCALING)
    E, F, _S, _h = pot(atoms)
    hf = pot.heat_flux
    ref = flux_oracle(family, atoms, atoms.get_velocities())
    vv = atoms.get_velocities()
    kin = (0.5 * atoms.get_masses() * (vv * vv).sum(1)) @ vv
    check_flux(hf["potential"], hf["convective"] - kin, ref, vv, f"{family} Potential_Dist")
    assert np.allclose(hf["total"], hf["potential"] + hf["convective"], rtol=0, atol=1e-14)
    calc = PESCalculator_Dist(potential=pot)
    assert "heat_flux" in calc.implemented_properties and "heat_flux" not in PESCalculator_Dist.implemented_properties
    calc.calculate(atoms, ["energy", "forces", "heat_flux"])
    assert np.abs(calc.results["heat_flux"] - hf["total"]).max() <= TOL_J_REL * ref["scale"] + 1e-12
    assert np.abs(calc.results["heat_flux_potential"] - hf["potential"]).max() <= TOL_J_REL * ref["scale"]
    # switched off between calls: the plain periodic evaluation, same energy
    pot.calc_heat_flux = False
    E2, F2, _S2, _ = pot(atoms)
    assert pot.heat_flux is None and abs(float(E2) - float(E)) <= 1e-8 * abs(float(E)) + 1e-7
    assert np.abs(F2.numpy() - F.numpy()).max() <= ftol(F.numpy())
    pot.calc_heat_flux = True
    # a few NVE steps that sample the flux at every force call; the last sample against the oracle
    md = MolecularDynamics(atoms, potential=pot, ensemble="nve", timestep=0.5)
    md.run(3)
    vv = md.atoms.get_velocities()
    ref = flux_oracle(family, md.atoms, vv)
    kin = (0.5 * md.atoms.get_masses() * (vv * vv).sum(1)) @ vv
    check_flux(pot.heat_flux["potential"], pot.heat_flux["convective"] - kin, ref, vv, f"{family} after 3 NVE steps")
    dm._engine.close()


# ------------------------------------------------------------- metamorphic, at sizes the oracle cannot reach
def flux_of(eng, model, atoms, v):
    set_structure(eng, model, atoms)
    _e, _f, _s, (j_pot, j_conv) = eng.compute_heat_flux(v)
    return j_pot, j_conv


# relative to max |J| over the components (J_pot sums terms of both signs, so its round-off is large against |J_pot|);
# observed on an H100: 1.5e-4 (TensorNet, doubled cell), 6.2e-5 (CHGNet)
TOL_SAME_J = 5e-4


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_permuting_the_atoms_leaves_the_flux(family):
    atoms = BIG[family]()
    model = model_of(family)
    v = velocities(len(atoms), 5)
    eng = engine_of(family, model)
    eng.set_heat_flux(reach_of(model))
    jp, jc = flux_of(eng, model, atoms, v)
    perm = np.random.default_rng(14).permutation(len(atoms))
    sym = np.array(atoms.get_chemical_symbols())[perm].tolist()
    jp2, jc2 = flux_of(eng, model, SimpleAtoms(sym, atoms.get_positions()[perm], atoms.get_cell()), v[perm])
    dp, dc = np.abs(jp2 - jp).max() / np.abs(jp).max(), np.abs(jc2 - jc).max() / np.abs(jc).max()
    print(f"{family} {len(atoms)} atoms, permuted: |dJ_pot| / |J_pot| {dp:.2e}, |dJ_conv| / |J_conv| {dc:.2e}; "
          f"{eng.counts()['n_own']} unfolded atoms")
    assert dp <= TOL_SAME_J and dc <= TOL_SAME_J
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_repeating_the_cell_doubles_the_flux(family):
    atoms = BIG[family]()
    model = model_of(family)
    v = velocities(len(atoms), 6)
    eng = engine_of(family, model)
    eng.set_heat_flux(reach_of(model))
    jp, jc = flux_of(eng, model, atoms, v)
    cell = np.array(atoms.get_cell())
    pos = atoms.get_positions()
    twice = SimpleAtoms(atoms.get_chemical_symbols() * 2, np.concatenate([pos, pos + cell[2]]),
                        cell * np.array([[1.0], [1.0], [2.0]]))
    jp2, jc2 = flux_of(eng, model, twice, np.concatenate([v, v]))
    # J_conv: each eps_i carries data_mean / N, which halves with twice the atoms
    jc2 = jc2 + SCALING["data_mean"] / len(atoms) * v.sum(0)
    dp, dc = np.abs(jp2 - 2 * jp).max() / np.abs(jp).max(), np.abs(jc2 - 2 * jc).max() / np.abs(jc).max()
    print(f"{family} {len(atoms)} atoms, cell twice along z: |dJ_pot| / |J_pot| {dp:.2e}, |dJ_conv| / |J_conv| {dc:.2e}")
    assert dp <= TOL_SAME_J and dc <= TOL_SAME_J
    eng.close()
