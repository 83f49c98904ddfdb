"""CPU, float64: the unfolded-cell heat flux of MACE (tests/mace_heat_flux_ref.py) for both hidden shapes (C x 0e and
C x 0e + C x 1o), without and with the ZBL pair term + Agnesi transform, on small models (C = 32, two interactions,
r_max 4.5 A: about 500 unfolded atoms for an 8-atom cell).

* the seeded form equals the definition sum_{i<n} sum_j r_ij (dU_i/dr_j . v_j) from the full Jacobian;
* finite differences of the barycentre B = sum_{i<n} r_i U_i along r + t v equal J_conv + J_pot - sum_j r_j (F~_j . v_j);
* J_pot does not depend on the centre c, nor on a translation of the whole structure followed by wrapping;
* at heat_flux_reach() = T r_max the cell atoms' energies, the folded forces and the energy equal the periodic ones and
  J is unchanged at reach + 3 A (also for a cell periodic along x and y only); at (T - 1) r_max they are not: the rule
  has no slack;
* every GPU tolerance of tests/test_gpu_mace_heat_flux.py is at least 10x below the error of the three bugs of
  oracle/heat_flux_ref.py, of the naive virial flux and of the two MACE-specific bugs;
* the wrapper's heat_flux_reach() is the oracle's, and MACECalculator_Dist advertises the flux only while it is on."""
import numpy as np
import pytest

from distmlip_b200.structures import SimpleAtoms, si_diamond
from oracle.mace_ref import potential_ref
from tests.mace_heat_flux_ref import barycentre, heat_flux_ref, reach_of
from tests.mace_zbl_ref import make_mace, make_mace_eq

TOL_J_REL = 1e-5  # tests/test_gpu_heat_flux.py, which tests/test_gpu_mace_heat_flux.py imports
SHAPES = {"0e": False, "0e+1o": True}
OPTIONS = {"plain": {}, "zbl+agnesi": dict(pair_repulsion=True, distance_transform="agnesi")}
CASES = [(s, o) for s in SHAPES for o in OPTIONS]


def model(shape, opt, seed=1, **kw):
    """the heat-flux tests' models: species Si and O, C = 32, two interactions, r_max 4.5 A, scale 8"""
    for k, v in dict(atomic_numbers=(14, 8), C=32, num_interactions=2, r_max=4.5, scale=8.0).items():
        kw.setdefault(k, v)
    return (make_mace_eq if SHAPES[shape] else make_mace)(seed=seed, **OPTIONS[opt], **kw)


def mixed(atoms, every=3):
    sym = ["O" if i % every == 0 else s for i, s in enumerate(atoms.get_chemical_symbols())]
    return SimpleAtoms(sym, atoms.get_positions(), np.array(atoms.get_cell()), pbc=atoms.get_pbc())


def cell8(seed=1):
    return mixed(si_diamond(1, sigma=0.15, seed=seed))


def squeezed8(seed=1):
    """cell8 at 0.85 of its size: Si-Si pairs inside the ZBL cutoff (2.22 A)"""
    a = cell8(seed)
    return SimpleAtoms(a.get_chemical_symbols(), 0.85 * a.get_positions(), 0.85 * np.array(a.get_cell()))


def slab8():
    """periodic along x and y only, 12 A of vacuum above and below"""
    a = cell8(5)
    cell = np.array(a.get_cell())
    cell[2, 2] = 30.0
    return SimpleAtoms(a.get_chemical_symbols(), a.get_positions() + [0, 0, 12.0], cell, pbc=(True, True, False))


def vel(n, seed=0):
    return np.random.default_rng(seed).normal(scale=0.05, size=(n, 3))


@pytest.mark.parametrize("shape,opt", CASES)
def test_seeded_form_equals_the_jacobian_definition(shape, opt):
    atoms = cell8()
    r = heat_flux_ref(model(shape, opt), atoms, vel(len(atoms)), jacobian=True)
    print(f"{shape} {opt}: {r['n_unfolded']} unfolded atoms, J_pot {r['j_pot']}, definition {r['j_pot_def']}")
    assert np.abs(r["j_pot"] - r["j_pot_def"]).max() <= 1e-10 * r["scale"]


@pytest.mark.parametrize("shape,opt", CASES)
def test_barycentre_derivative(shape, opt):
    atoms = cell8(2)
    v = vel(len(atoms), 1)
    m = model(shape, opt)
    r = heat_flux_ref(m, atoms, v)
    h = 1e-2
    B = barycentre(m, atoms, v, [-2 * h, -h, h, 2 * h])
    dB = (B[0] - 8 * B[1] + 8 * B[2] - B[3]) / (12 * h)
    vu = v[r["image_of"]]
    rhs = r["j_conv"] + r["j_pot"] - (r["unfolded"] * np.einsum("jk,jk->j", r["forces_unfolded"], vu)[:, None]).sum(0)
    print(f"{shape} {opt}: dB/dt {dB}, J_conv + J_pot - sum r (F.v) {rhs}")
    assert np.abs(dB - rhs).max() <= 1e-8 * np.abs(rhs).max()


@pytest.mark.parametrize("shape,opt", CASES)
def test_centre_and_translation_do_not_change_j_pot(shape, opt):
    atoms = cell8(3)
    v = vel(len(atoms), 2)
    m = model(shape, opt)
    r0 = heat_flux_ref(m, atoms, v)
    r1 = heat_flux_ref(m, atoms, v, centre=np.array([3.0, -2.0, 7.5]))
    assert np.abs(r1["j_pot"] - r0["j_pot"]).max() <= 1e-10 * r0["scale"]
    cell = np.array(atoms.get_cell())
    wrapped = ((atoms.get_positions() + np.array([2.1, -0.7, 4.4])) @ np.linalg.inv(cell) % 1.0) @ cell
    r2 = heat_flux_ref(m, SimpleAtoms(atoms.get_chemical_symbols(), wrapped, cell), v)
    print(f"{shape} {opt}: J_pot {r0['j_pot']}, centre moved {r1['j_pot']}, translated + wrapped {r2['j_pot']}")
    assert np.abs(r2["j_pot"] - r0["j_pot"]).max() <= 1e-10 * r0["scale"]
    assert np.abs(r2["j_conv"] - r0["j_conv"]).max() <= 1e-12


@pytest.mark.parametrize("cell", ["cell8", "slab8"])
@pytest.mark.parametrize("shape,opt", CASES)
def test_reach_reproduces_the_periodic_values_and_has_no_slack(shape, opt, cell):
    atoms = {"cell8": cell8, "slab8": slab8}[cell]()
    m = model(shape, opt)
    v = vel(len(atoms), 3)
    E, F, _S, eps = potential_ref(m, atoms)
    r = heat_flux_ref(m, atoms, v)
    assert abs(r["energy"] - E.item()) <= 1e-10 * abs(E.item())
    assert np.abs(r["energies"] - eps.numpy()).max() <= 1e-10
    assert np.abs(r["forces"] - F.numpy()).max() <= 1e-10
    wider = heat_flux_ref(m, atoms, v, reach=reach_of(m) + 3.0)
    print(f"{shape} {opt} {cell}: {r['n_unfolded']} -> {wider['n_unfolded']} unfolded atoms; J_pot {r['j_pot']} / "
          f"{wider['j_pot']}")
    assert np.abs(wider["j_pot"] - r["j_pot"]).max() <= 1e-10 * r["scale"]
    assert np.abs(wider["j_conv"] - r["j_conv"]).max() <= 1e-12
    # one hop short: the outermost cell atoms miss part of their receptive field
    T = len(m.interactions)
    short = heat_flux_ref(m, atoms, v, reach=(T - 1) * float(m.r_max))
    de, df = np.abs(short["energies"] - eps.numpy()).max(), np.abs(short["forces"] - F.numpy()).max()
    print(f"{shape} {opt} {cell}: at (T - 1) r_max max |d eps| {de:.2e} eV, max |dF| {df:.2e} eV/A")
    assert de > 1e-7 and df > 1e-7


@pytest.mark.parametrize("shape,opt", CASES)
def test_naive_virial_flux_differs_and_gpu_tolerances_see_the_bugs(shape, opt):
    atoms = squeezed8()
    r = heat_flux_ref(model(shape, opt), atoms, vel(len(atoms)), naive=True, mutants=True)
    jp = r["j_pot"]
    rel = np.linalg.norm(r["j_naive"] - jp) / np.linalg.norm(jp)
    print(f"{shape} {opt}: |J_naive - J_pot| / |J_pot| = {rel:.3f}")
    assert rel >= 0.02
    tol = TOL_J_REL * r["scale"]
    errs = {name: np.abs(j - jp).max() for name, j in r["mutants"].items()}
    errs["naive"] = np.abs(r["j_naive"] - jp).max()
    print(f"{shape} {opt}: GPU tolerance {tol:.2e}; bug errors", {k: f"{e:.2e}" for k, e in errs.items()})
    assert "readout_adjoint_unweighted" in errs and ("zbl_unweighted" in errs) == (opt != "plain")
    for name, e in errs.items():
        assert e >= 10 * tol, (name, e, tol)


@pytest.mark.parametrize("shape,opt", CASES)
def test_wrapper_reach_is_the_oracle_reach(shape, opt):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    for T, r_max in ((2, 4.5), (3, 5.3)):
        m = model(shape, opt, num_interactions=T, r_max=r_max)
        assert ScaleShiftMACE_Dist.from_existing(m).heat_flux_reach() == reach_of(m) == T * r_max


def test_calculator_advertises_the_flux_only_while_it_is_on():
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    class Calc:  # the attribute surface of mace's MACECalculator
        def __init__(self, models):
            self.models, self.r_max = models, 4.5

    flux = ("heat_flux", "heat_flux_potential")
    one = MACECalculator_Dist.from_existing(Calc([model("0e", "plain")]))
    assert not one.calc_heat_flux and not set(flux) & set(one.implemented_properties)
    on = MACECalculator_Dist.from_existing(Calc([model("0e", "plain")]), calc_heat_flux=True, heat_flux_reach=12.0)
    assert set(flux) <= set(on.implemented_properties) and on.heat_flux_reach == 12.0
    assert not set(flux) & set(MACECalculator_Dist.implemented_properties)
    on.calc_heat_flux = False
    assert not set(flux) & set(on.implemented_properties) and "forces" in on.implemented_properties
    committee = MACECalculator_Dist.from_existing(Calc([model("0e", "plain"), model("0e+1o", "zbl+agnesi")]))
    committee.calc_heat_flux = True
    assert set(flux) | {"energies", "forces_comm"} <= set(committee.implemented_properties)
