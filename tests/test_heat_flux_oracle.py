"""CPU, float64: the unfolded-cell heat flux of oracle/heat_flux_ref.py, for CHGNet and TensorNet.

* the seeded form equals the definition sum_{i<n} sum_j r_ij (dU_i/dr_j . v_j) from the full Jacobian;
* finite differences of the barycentre B = sum_{i<n} r_i U_i along r + t v equal J_conv,pot + J_pot - sum_j r_j (F~_j . v_j);
* J_pot does not depend on the centre c, nor on a translation of the whole structure followed by wrapping;
* at the model's heat_flux_reach the cell atoms' energies, the folded forces and J_pot equal the periodic values (and J
  at reach + 3 A), also for a cell periodic along x and y only;
* the naive virial flux -sum_i w_i v_i differs from J_pot: the reason the feature exists;
* every GPU tolerance of tests/test_gpu_heat_flux.py is at least 10x below the error of four plausible bugs."""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, si_diamond
from oracle.atomic_ref import atomic_ref
from oracle.heat_flux_ref import barycentre, heat_flux_ref, reach_of
from tests._util import make_model
from tests.test_oracle_tensornet import make_tn

SCALING = dict(data_mean=0.7, data_std=1.3)
TOL_J_REL = 1e-5  # tests/test_gpu_heat_flux.py


def model_of(family):
    return make_model(seed=2) if family == "chgnet" else make_tn(seed=3, scale=1.5)


def refs(model):
    return np.linspace(-0.5, 0.5, len(model.element_types))


def cell8(seed=1):
    a = si_diamond(1, sigma=0.15, seed=seed)
    sym = ["O" if i % 3 == 0 else s for i, s in enumerate(a.get_chemical_symbols())]
    return SimpleAtoms(sym, a.get_positions(), a.get_cell())


def cell16():
    a = si_diamond(1, sigma=0.15, seed=4, nz=2)
    sym = ["Ge" if i % 2 == 0 else s for i, s in enumerate(a.get_chemical_symbols())]
    return SimpleAtoms(sym, a.get_positions(), a.get_cell())


def slab8():
    """periodic along x and y only, 12 A of vacuum above and below"""
    a = cell8(5)
    cell = np.array(a.get_cell())
    cell[2, 2] = 30.0
    return SimpleAtoms(a.get_chemical_symbols(), a.get_positions() + [0, 0, 12.0], cell, pbc=(True, True, False))


def vel(n, seed=0):
    return np.random.default_rng(seed).normal(scale=0.05, size=(n, 3))


def flux(family, atoms, v, **kw):
    model = model_of(family)
    return heat_flux_ref(model, atoms, v, element_refs=refs(model), **SCALING, **kw)


FAMILIES = ["chgnet", "tensornet"]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("cell", ["cell8", "cell16"])
def test_seeded_form_equals_the_jacobian_definition(family, cell):
    atoms = {"cell8": cell8, "cell16": cell16}[cell]()
    r = flux(family, atoms, vel(len(atoms)), jacobian=True)
    print(f"{family} {cell}: {r['n_unfolded']} unfolded atoms, J_pot {r['j_pot']}, definition {r['j_pot_def']}")
    assert np.abs(r["j_pot"] - r["j_pot_def"]).max() <= 1e-10 * r["scale"]


@pytest.mark.parametrize("family", FAMILIES)
def test_barycentre_derivative(family):
    atoms = cell8(2)
    v = vel(len(atoms), 1)
    model = model_of(family)
    r = flux(family, atoms, v)
    h = 1e-2
    B = barycentre(model, atoms, v, [-2 * h, -h, h, 2 * h], data_std=SCALING["data_std"])
    dB = (B[0] - 8 * B[1] + 8 * B[2] - B[3]) / (12 * h)
    n = len(atoms)
    j_conv_pot = ((r["energies"] - refs(model)[[model.element_types.index(s) for s in atoms.get_chemical_symbols()]]
                   - SCALING["data_mean"] / n)[:, None] * v).sum(0)
    vu = v[r["image_of"]]
    rhs = j_conv_pot + r["j_pot"] - (r["unfolded"] * np.einsum("jk,jk->j", r["forces_unfolded"], vu)[:, None]).sum(0)
    print(f"{family}: dB/dt {dB}, J_conv,pot + J_pot - sum r (F.v) {rhs}")
    assert np.abs(dB - rhs).max() <= 1e-8 * np.abs(rhs).max()


@pytest.mark.parametrize("family", FAMILIES)
def test_centre_and_translation_do_not_change_j_pot(family):
    atoms = cell8(3)
    v = vel(len(atoms), 2)
    r0 = flux(family, atoms, v)
    r1 = flux(family, atoms, v, centre=np.array([3.0, -2.0, 7.5]))
    assert np.abs(r1["j_pot"] - r0["j_pot"]).max() <= 1e-10 * r0["scale"]
    cell = np.array(atoms.get_cell())
    moved = atoms.get_positions() + np.array([2.1, -0.7, 4.4])
    frac = moved @ np.linalg.inv(cell)
    wrapped = (frac % 1.0) @ cell
    r2 = flux(family, SimpleAtoms(atoms.get_chemical_symbols(), wrapped, cell), v)
    print(f"{family}: J_pot {r0['j_pot']}, centre moved {r1['j_pot']}, translated + wrapped {r2['j_pot']}")
    assert np.abs(r2["j_pot"] - r0["j_pot"]).max() <= 1e-10 * r0["scale"]
    assert np.abs(r2["j_conv"] - r0["j_conv"]).max() <= 1e-12


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("cell", ["cell8", "slab8"])
def test_reach_reproduces_the_periodic_values(family, cell):
    atoms = {"cell8": cell8, "slab8": slab8}[cell]()
    model = model_of(family)
    v = vel(len(atoms), 3)
    r = flux(family, atoms, v)
    per = atomic_ref(model, atoms, element_refs=refs(model), dtype=torch.float64, **SCALING)
    assert abs(r["energy"] - float(per["energy"])) <= 1e-10 * abs(float(per["energy"]))
    assert np.abs(r["energies"] - per["energies"].numpy()).max() <= 1e-10
    assert np.abs(r["forces"] - per["forces"].numpy()).max() <= 1e-10
    wider = flux(family, atoms, v, reach=reach_of(model) + 3.0)
    print(f"{family} {cell}: {r['n_unfolded']} -> {wider['n_unfolded']} unfolded atoms; J_pot {r['j_pot']} / "
          f"{wider['j_pot']}")
    assert np.abs(wider["j_pot"] - r["j_pot"]).max() <= 1e-10 * r["scale"]
    assert np.abs(wider["j_conv"] - r["j_conv"]).max() <= 1e-12


@pytest.mark.parametrize("family", FAMILIES)
def test_naive_virial_flux_differs_and_gpu_tolerances_see_the_bugs(family):
    atoms = cell8(1)
    r = flux(family, atoms, vel(len(atoms)), naive=True, mutants=True)
    jp = r["j_pot"]
    rel = np.linalg.norm(r["j_naive"] - jp) / np.linalg.norm(jp)
    print(f"{family}: |J_naive - J_pot| / |J_pot| = {rel:.3f}")
    assert rel >= 0.02
    tol = TOL_J_REL * r["scale"]
    errs = {name: np.abs(j - jp).max() for name, j in r["mutants"].items()}
    errs["naive"] = np.abs(r["j_naive"] - jp).max()
    print(f"{family}: GPU tolerance {tol:.2e}; bug errors", {k: f"{e:.2e}" for k, e in errs.items()})
    for name, e in errs.items():
        assert e >= 10 * tol, (name, e, tol)
