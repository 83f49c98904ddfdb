"""GPU: the heat flux of MACE (ScaleShiftMACE_Dist.evaluate_heat_flux, MACECalculator_Dist(calc_heat_flux=True);
DESIGN.md §10) for both hidden shapes, without and with the ZBL pair term + Agnesi transform, against the float64
unfolded-cell oracle (tests/mace_heat_flux_ref.py); the unfolded evaluation against a plain periodic handle; partition
independence in single-process groups; the off -> on -> off round trip; the calculator (one model, a committee, other
energy units, NVE steps); and, beyond the oracle's reach, invariance under a permutation of the atoms and additivity
under a repeat of the cell.

The tolerances are those of tests/test_gpu_heat_flux.py; tests/test_heat_flux_oracle_mace.py checks that they stay at
least 10x below the error of plausible bugs, the two MACE-specific ones included."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
try:
    import ase  # noqa: F401
except ImportError:
    sys.path.insert(0, os.path.join(HERE, "stubs"))
    import ase  # noqa: F401

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.mace_ref import atomic_virials_ref
from tests.mace_heat_flux_ref import heat_flux_ref, reach_of
from tests.test_gpu_heat_flux import TOL_J_REL, TOL_JCONV, TOL_SAME_J, velocities
from tests.test_heat_flux_oracle_mace import CASES, mixed, model

pytestmark = pytest.mark.gpu


def check_flux(j_pot, j_conv, ref, v, what=""):
    """tests/test_gpu_heat_flux.py check_flux; J_conv per unit of sum_i |v_i| within TOL_JCONV or, where the ZBL pair
    energies of close contacts make eps_i large, 2e-7 of max |eps_i| (the fp32 round-off of eps_i)"""
    dp = np.abs(j_pot - ref["j_pot"]).max() / ref["scale"]
    dc = np.abs(j_conv - ref["j_conv"]).max() / np.abs(v).sum()
    tc = max(TOL_JCONV, 2e-7 * np.abs(ref["energies"]).max())
    print(f"heat flux {what}: |dJ_pot| / scale {dp:.2e} (scale {ref['scale']:.3e}), |dJ_conv| / sum|v| {dc:.2e} eV "
          f"(tolerance {tc:.1e}, max |eps| {np.abs(ref['energies']).max():.1f} eV)")
    assert dp <= TOL_J_REL, dp
    assert dc <= tc, dc


def wrapper(m, gpus=(0,)):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode(list(gpus))
    return d


def ftol(f0):
    """fp32 forces of two graphs of the same structure (edge order, atomics, the fold)"""
    return 1e-6 * float(np.abs(f0).max()) + 1e-5


STRUCTURES = {
    "diamond64": lambda: mixed(si_diamond(2, sigma=0.15, seed=1)),
    "rough": lambda: mixed(rough_cell(100, min_dist=0.7, seed=3), every=2),  # close contacts: the ZBL term at work
}


@pytest.mark.parametrize("structure", list(STRUCTURES))
@pytest.mark.parametrize("shape,opt", CASES)
def test_flux_matches_the_oracle(shape, opt, structure):
    atoms = STRUCTURES[structure]()
    m = model(shape, opt, seed=2)
    v = velocities(len(atoms), 1)
    d = wrapper(m)
    e, f, _s, _ae, _av, (j_pot, j_conv) = d.evaluate_heat_flux(atoms, v)
    ref = heat_flux_ref(m, atoms, v)
    c = d._engine.counts()
    print(f"{shape} {opt} {structure}: {len(atoms)} atoms -> {c['n_own']} unfolded, {c['n_edges']} edges "
          f"(oracle {ref['n_unfolded']}, {ref['n_edges']})")
    if structure == "diamond64":
        assert c["n_own"] == ref["n_unfolded"] and c["n_edges"] == ref["n_edges"]
    check_flux(j_pot, j_conv, ref, v, f"{shape} {opt} {structure}")
    assert abs(e - ref["energy"]) / len(atoms) <= 1e-4 + 1e-6 * np.abs(ref["energies"]).max()
    assert np.abs(f - ref["forces"]).max() <= 1e-3 + 1e-5 * np.abs(ref["forces"]).max()
    d._engine.close()


@pytest.mark.parametrize("shape,opt", CASES)
def test_unfolded_evaluation_equals_the_periodic_one(shape, opt):
    atoms = STRUCTURES["rough"]()
    m = model(shape, opt, seed=3)
    plain = wrapper(m)
    e0, f0, s0, eps0, w0 = plain.evaluate(atoms, atomic=True)
    d = wrapper(m)
    e1, f1, s1, eps1, w1, _j = d.evaluate_heat_flux(atoms, velocities(len(atoms)), atomic=True)
    de, df, ds = abs(e1 - e0), np.abs(f1 - f0).max(), np.abs(s1 - s0).max()
    deps, dw = np.abs(eps1 - eps0).max(), np.abs(w1 - w0).max() / np.abs(w0).max()
    print(f"unfolded vs periodic {shape} {opt}: |dE| {de:.2e} eV, |dF| {df:.2e} eV/A (max |F| {np.abs(f0).max():.2f}), "
          f"|dS| {ds:.2e} GPa, |d eps| {deps:.2e} eV, |dw| / max|w| {dw:.2e}")
    assert de <= 1e-6 * np.abs(eps0).sum() + 1e-5
    assert df <= ftol(f0), df
    assert ds <= 1e-5 * np.abs(s0).max() + 1e-5, ds
    assert deps <= 1e-5 + 2e-7 * np.abs(eps0).max() and dw <= 1e-5
    # per-atom virials of the masked pass against the oracle as well: the ZBL term belongs to dst
    w_ref = atomic_virials_ref(m, atoms).numpy()
    assert np.abs(w1 - w_ref).max() <= 1e-4 * max(1.0, np.abs(w_ref).max())
    plain._engine.close()
    d._engine.close()


@pytest.mark.parametrize("parts", [2, 3])
def test_partitions_of_a_group_give_the_same_flux(parts):
    atoms = mixed(si_diamond(2, sigma=0.15, seed=5, nz=12))  # 65 A along z: slabs wider than the reach
    m = model("0e+1o", "zbl+agnesi", seed=4)
    v = velocities(len(atoms), 3)
    one = wrapper(m)
    e1, f1, _s1, _a1, _w1, (jp1, jc1) = one.evaluate_heat_flux(atoms, v)
    grp = wrapper(m, [0] * parts)
    e2, f2, _s2, _a2, _w2, (jp2, jc2) = grp.evaluate_heat_flux(atoms, v)
    assert grp._engine.counts()["world"] == parts
    dp, dc = np.abs(jp2 - jp1).max() / np.abs(jp1).max(), np.abs(jc2 - jc1).max() / np.abs(jc1).max()
    print(f"{parts} partitions vs 1: |dJ_pot| / |J_pot| {dp:.2e}, |dJ_conv| / |J_conv| {dc:.2e}, "
          f"|dF| {np.abs(f2 - f1).max():.2e}")
    assert dp <= TOL_SAME_J and dc <= TOL_SAME_J
    assert abs(e2 - e1) / len(atoms) <= 1e-6 and np.abs(f2 - f1).max() <= ftol(f1)
    one._engine.close()
    grp._engine.close()


def test_off_on_off_on_one_handle():
    atoms = STRUCTURES["diamond64"]()
    m = model("0e+1o", "zbl+agnesi", seed=5)
    d = wrapper(m)
    eng = d._engine
    e0, f0, s0, _, _ = d.evaluate(atoms)
    launches_off = eng.counts()["launches"]
    with pytest.raises(ValueError):
        d.evaluate_heat_flux(atoms, velocities(len(atoms)), reach=reach_of(m) - 0.5)
    e1, f1, s1, _, _, _j = d.evaluate_heat_flux(atoms, velocities(len(atoms)))
    assert eng.counts()["n_own"] > len(atoms)
    e2, f2, s2, _, _ = d.evaluate(atoms)
    assert eng.counts()["launches"] == launches_off
    assert eng.counts()["n_own"] == len(atoms)
    for e, f, s in ((e1, f1, s1), (e2, f2, s2)):
        assert abs(e - e0) <= 1e-7 * abs(e0) + 1e-5
        assert np.abs(f - f0).max() <= ftol(f0), (np.abs(f - f0).max(), ftol(f0))
        assert np.abs(s - s0).max() <= 1e-5 * np.abs(s0).max() + 1e-5
    eng.close()


class Moving:
    """SimpleAtoms with velocities and masses, for the calculator"""

    def __init__(self, a, v):
        self.a, self.v = a, v

    def __getattr__(self, name):
        return getattr(self.a, name)

    def __len__(self):
        return len(self.a)

    def get_velocities(self):
        return self.v.copy()

    def get_masses(self):
        return np.where(np.array(self.a.get_chemical_symbols()) == "O", 15.999, 28.085)


class Calc:  # the attribute surface of mace's MACECalculator
    def __init__(self, models, energy_units_to_eV=1.0):
        self.models, self.r_max = models, 4.5
        self.energy_units_to_eV, self.length_units_to_A = energy_units_to_eV, 1.0


def kinetic(atoms):
    v = atoms.get_velocities()
    return (0.5 * atoms.get_masses() * (v * v).sum(1)) @ v


def test_calculator_single_and_committee():
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    base = STRUCTURES["rough"]()
    atoms = Moving(base, velocities(len(base), 4))
    v = atoms.get_velocities()
    ms = [model("0e", "plain", seed=11), model("0e+1o", "zbl+agnesi", seed=12)]
    refs = [heat_flux_ref(m, base, v) for m in ms]
    calc = MACECalculator_Dist.from_existing(Calc(ms[:1]), calc_heat_flux=True)
    calc.enable_distributed_mode([0])
    calc.calculate(atoms)
    r = calc.results
    assert "heat_flux" in calc.implemented_properties
    check_flux(r["heat_flux_potential"], r["heat_flux"] - r["heat_flux_potential"] - kinetic(atoms), refs[0], v,
               "calculator, one model")
    e_single = r["energy"]
    # switched off between calls: the plain periodic evaluation, the same energy, no flux
    calc.calc_heat_flux = False
    calc.calculate(atoms)
    assert "heat_flux" not in calc.results and "heat_flux" not in calc.implemented_properties
    assert abs(calc.results["energy"] - e_single) <= 1e-7 * abs(e_single) + 1e-5
    # a committee in other energy units: eps and J_pot scale with the energy, the kinetic term does not
    com = MACECalculator_Dist.from_existing(Calc(ms, energy_units_to_eV=2.0), calc_heat_flux=True)
    com.enable_distributed_mode([0])
    com.calculate(atoms)
    r = com.results
    want_pot = 2.0 * np.mean([x["j_pot"] for x in refs], axis=0)
    want_conv = 2.0 * np.mean([x["j_conv"] for x in refs], axis=0)
    scale = 2.0 * max(x["scale"] for x in refs)
    dp = np.abs(r["heat_flux_potential"] - want_pot).max() / scale
    dc = np.abs(r["heat_flux"] - r["heat_flux_potential"] - kinetic(atoms) - want_conv).max() / np.abs(v).sum()
    print(f"committee, energy_units_to_eV = 2: |dJ_pot| / scale {dp:.2e}, |dJ_conv| / sum|v| {dc:.2e}")
    assert dp <= TOL_J_REL and dc <= 2.0 * max(TOL_JCONV, 2e-7 * max(np.abs(x["energies"]).max() for x in refs))
    assert abs(r["energy"] - 2.0 * np.mean([x["energy"] for x in refs])) / len(base) <= 2e-4
    for m in calc.models + com.models:
        m._engine.close()


def test_calculator_nve_steps():
    from ase import Atoms

    from distmlip_b200.implementations.matgl import MolecularDynamics
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    # silicon only, as the ASE stand-in reports Z = 14
    base = si_diamond(2, sigma=0.15, seed=8)
    atoms = Atoms(symbols=base.get_chemical_symbols(), positions=base.get_positions(), cell=base.get_cell(), pbc=True)
    atoms.set_momenta(velocities(len(atoms), 5) * atoms.get_masses()[:, None])
    m = model("0e+1o", "zbl+agnesi", seed=13)
    calc = MACECalculator_Dist.from_existing(Calc([m]), calc_heat_flux=True)
    calc.enable_distributed_mode([0])
    md = MolecularDynamics(atoms, potential=calc, ensemble="nve", timestep=0.5)
    md.run(3)
    vv = md.atoms.get_velocities()
    sym = SimpleAtoms(md.atoms.get_chemical_symbols(), md.atoms.get_positions(), md.atoms.get_cell())
    ref = heat_flux_ref(m, sym, vv)
    r = calc.results
    check_flux(r["heat_flux_potential"], r["heat_flux"] - r["heat_flux_potential"] - kinetic(md.atoms), ref, vv,
               "after 3 NVE steps")
    calc.models[0]._engine.close()


# ------------------------------------------------------------- metamorphic, at sizes the oracle cannot reach
BIG = lambda: mixed(si_diamond(12, sigma=0.15, seed=13))  # noqa: E731  13 824 atoms


def test_permuting_the_atoms_leaves_the_flux():
    atoms = BIG()
    d = wrapper(model("0e+1o", "zbl+agnesi", seed=6))
    v = velocities(len(atoms), 5)
    *_, (jp, jc) = d.evaluate_heat_flux(atoms, v)
    perm = np.random.default_rng(14).permutation(len(atoms))
    sym = np.array(atoms.get_chemical_symbols())[perm].tolist()
    *_, (jp2, jc2) = d.evaluate_heat_flux(SimpleAtoms(sym, atoms.get_positions()[perm], atoms.get_cell()), v[perm])
    dp, dc = np.abs(jp2 - jp).max() / np.abs(jp).max(), np.abs(jc2 - jc).max() / np.abs(jc).max()
    print(f"{len(atoms)} atoms, permuted: |dJ_pot| / |J_pot| {dp:.2e}, |dJ_conv| / |J_conv| {dc:.2e}; "
          f"{d._engine.counts()['n_own']} unfolded atoms, {d._engine.counts()['n_edges']} edges")
    assert dp <= TOL_SAME_J and dc <= TOL_SAME_J
    d._engine.close()


def test_repeating_the_cell_doubles_the_flux():
    atoms = BIG()
    d = wrapper(model("0e+1o", "zbl+agnesi", seed=6))
    v = velocities(len(atoms), 6)
    *_, (jp, jc) = d.evaluate_heat_flux(atoms, v)
    cell = np.array(atoms.get_cell())
    pos = atoms.get_positions()
    twice = SimpleAtoms(atoms.get_chemical_symbols() * 2, np.concatenate([pos, pos + cell[2]]),
                        cell * np.array([[1.0], [1.0], [2.0]]))
    *_, (jp2, jc2) = d.evaluate_heat_flux(twice, np.concatenate([v, v]))
    dp, dc = np.abs(jp2 - 2 * jp).max() / np.abs(jp).max(), np.abs(jc2 - 2 * jc).max() / np.abs(jc).max()
    print(f"{len(atoms)} atoms, cell twice along z: |dJ_pot| / |J_pot| {dp:.2e}, |dJ_conv| / |J_conv| {dc:.2e}")
    assert dp <= TOL_SAME_J and dc <= TOL_SAME_J
    d._engine.close()
