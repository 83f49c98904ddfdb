"""GPU: per-atom energies and per-atom virials (b2m_set_atomic / b2m_get_atomic) of CHGNet and TensorNet against the
autograd oracle (oracle/atomic_ref.py), their sum rules against the engine's own energy and stress, partition
independence in single-process groups, the off -> on -> off round trip on one handle, and PESCalculator_Dist."""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.atomic_ref import atomic_ref
from tests._util import engine_from_model, make_model
from tests.test_gpu_tensornet import tn_engine
from tests.test_oracle_tensornet import make_tn

pytestmark = pytest.mark.gpu
GPA_PER_EVA3 = 160.21766208
B2M_ERR_STATE = -6
TOL_EPS = 1e-4  # eV per atom
TOL_W = 5e-3    # eV per virial component (1e-3 eV/A force tolerance x 5 A cutoff)
SCALING = dict(data_mean=0.7, data_std=1.3)


def mixed(atoms, other="O", every=3):
    sym = [other if i % every == 0 else s for i, s in enumerate(atoms.get_chemical_symbols())]
    return SimpleAtoms(sym, atoms.get_positions(), atoms.get_cell())


def model_of(family):
    return make_model(seed=2) if family == "chgnet" else make_tn(seed=3, scale=1.5)


def refs(model):
    return np.linspace(-0.5, 0.5, len(model.element_types))


def engine_of(family, model, device=0):
    make = engine_from_model if family == "chgnet" else tn_engine
    return make(model, device=device, element_refs=refs(model), **SCALING)


def set_structure(eng, model, atoms):
    sp = np.array([model.element_types.index(s) for s in atoms.get_chemical_symbols()], dtype=np.int32)
    eng.set_structure(atoms.get_positions(), np.array(atoms.get_cell()), sp, atoms.get_pbc().astype(np.int32))


def oracle(family, atoms):
    model = model_of(family)
    return atomic_ref(model, atoms, element_refs=refs(model), dtype=torch.float64, **SCALING)


def check_against_oracle(eps, w, ref):
    de = np.abs(eps - ref["energies"].numpy()).max()
    dw = np.abs(w - ref["virials"].numpy()).max()
    assert de < TOL_EPS, de
    assert dw < TOL_W, (dw, np.abs(ref["virials"].numpy()).max())


def check_sum_rules(eps, w, e, s, volume):
    assert abs(eps.sum() - e) <= 1e-6 * abs(e), (eps.sum(), e)
    sig = w.astype(np.float64).sum(0) / volume * GPA_PER_EVA3
    assert np.abs(sig - s).max() <= 1e-5 * np.abs(s).max() + 1e-6, (sig, s)


STRUCTURES = {
    "diamond64": lambda: mixed(si_diamond(2, sigma=0.15, seed=1)),
    "diamond512": lambda: mixed(si_diamond(4, sigma=0.15, seed=2)),
    "rough": lambda: mixed(rough_cell(300, seed=4), other="Ge", every=2),
}


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("structure", list(STRUCTURES))
def test_per_atom_values_match_the_oracle(family, structure):
    atoms = STRUCTURES[structure]()
    model = model_of(family)
    eng = engine_of(family, model)
    set_structure(eng, model, atoms)
    eng.set_atomic(True)
    e, _f, s = eng.compute(forces=True, stress=True)
    eps, w = eng.atomic()
    assert eps.dtype == np.float64 and eps.shape == (len(atoms),)
    assert w.dtype == np.float32 and w.shape == (len(atoms), 3, 3)
    check_against_oracle(eps, w, oracle(family, atoms))
    check_sum_rules(eps, w, e, s, atoms.get_volume())
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_partitions_of_a_group_give_the_same_per_atom_values(family):
    atoms = mixed(si_diamond(2, sigma=0.15, seed=5, nz=12))  # three 21.7 A slabs
    model = model_of(family)
    ref = oracle(family, atoms)
    got = []
    for devs in ([0], [0, 0], [0, 0, 0]):
        eng = engine_of(family, model, device=devs)
        set_structure(eng, model, atoms)
        eng.set_atomic(True)
        e, _f, s = eng.compute(forces=True, stress=True)
        assert eng.counts()["world"] == len(devs)
        eps, w = eng.atomic()
        check_against_oracle(eps, w, ref)
        check_sum_rules(eps, w, e, s, atoms.get_volume())
        got.append((eps, w))
        eng.close()
    wmax = max(1.0, float(np.abs(got[0][1]).max()))
    for eps, w in got[1:]:  # fp32 atomics in a different order: round-off level
        assert np.abs(eps - got[0][0]).max() < 1e-5
        assert np.abs(w - got[0][1]).max() < 2e-5 * wmax


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_off_on_off_on_one_handle(family):
    from distmlip_b200._lib import B2MError

    atoms = mixed(si_diamond(3, sigma=0.15, seed=6))
    model = model_of(family)
    eng = engine_of(family, model)
    set_structure(eng, model, atoms)
    e0, f0, s0 = eng.compute()
    launches_off = eng.counts()["launches"]
    _e, f0b, _s = eng.compute()
    print(f"off -> off: max |dF| {np.abs(f0b - f0).max():.2e} eV/A (fp32 atomic order)")
    with pytest.raises(B2MError) as ei:
        eng.atomic()
    assert ei.value.code == B2M_ERR_STATE
    eng.set_atomic(True)
    e1, f1, s1 = eng.compute()
    eps, w = eng.atomic()
    check_sum_rules(eps, w, e1, s1, atoms.get_volume())
    # energy only: energies exist, virials do not
    e_only, _, _ = eng.compute(forces=False, stress=False)
    eps2, none = eng.atomic(virials=False)
    assert none is None and abs(eps2.sum() - e_only) <= 1e-6 * abs(e_only)
    assert np.abs(eps2 - eps).max() < 1e-5
    with pytest.raises(B2MError) as ei:
        eng.atomic()
    assert ei.value.code == B2M_ERR_STATE
    eng.set_atomic(False)
    e2, f2, s2 = eng.compute()
    assert eng.counts()["launches"] == launches_off
    with pytest.raises(B2MError) as ei:
        eng.atomic(virials=False)
    assert ei.value.code == B2M_ERR_STATE
    # forces: 1e-8 relative, or 5e-8 eV/A where the forces are small (the fp32 atomics of the force scatter alone move
    # them by ~1e-8 eV/A between two evaluations in the off state)
    ftol = max(1e-8 * float(np.abs(f0).max()), 5e-8)
    for e, f in ((e1, f1), (e2, f2)):
        assert abs(e - e0) <= 1e-8 * abs(e0)
        assert np.abs(f - f0).max() <= ftol, (np.abs(f - f0).max(), ftol)
    eng.close()


def test_release_workspace_drops_the_per_atom_results():
    from distmlip_b200._lib import B2MError

    atoms = mixed(si_diamond(2, sigma=0.15, seed=7))
    model = model_of("chgnet")
    eng = engine_of("chgnet", model)
    eng.set_atomic(True)
    set_structure(eng, model, atoms)
    eng.compute()
    eng.atomic()
    eng.release_workspace()
    set_structure(eng, model, atoms)
    with pytest.raises(B2MError) as ei:
        eng.atomic()
    assert ei.value.code == B2M_ERR_STATE
    e, _f, s = eng.compute()  # the flag survives the release: buffers come back on the next evaluation
    eps, w = eng.atomic()
    check_sum_rules(eps, w, e, s, atoms.get_volume())
    eng.close()


@pytest.mark.parametrize("family,devices", [("chgnet", [0]), ("tensornet", [0, 0])])
def test_calculator_end_to_end(family, devices):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, PESCalculator_Dist, Potential_Dist, TensorNet_Dist

    atoms = mixed(si_diamond(2, sigma=0.15, seed=8, nz=8))
    model = model_of(family)
    dm = (CHGNet_Dist if family == "chgnet" else TensorNet_Dist).from_existing(model)
    dm.enable_distributed_mode(devices)
    pot = Potential_Dist(model=dm, element_refs=refs(model), calc_atomic=True, **SCALING)
    out = pot(atoms)
    assert len(out) == 4
    E, _F, S, _h = out
    assert pot.atomic_energies.dtype == torch.float64 and pot.atomic_stresses.dtype == torch.float32
    assert pot.atomic_stresses.shape == (len(atoms), 3, 3)
    assert abs(float(pot.atomic_energies.sum()) - float(E)) <= 1e-6 * abs(float(E))
    sig = pot.atomic_stresses.double().sum(0)
    assert float((sig - S.double()).abs().max()) <= 1e-5 * float(S.abs().max()) + 1e-6
    ref = oracle(family, atoms)
    check_against_oracle(pot.atomic_energies.numpy(), pot.atomic_stresses.numpy() * atoms.get_volume() / GPA_PER_EVA3,
                         ref)
    for use_voigt in (False, True):
        calc = PESCalculator_Dist(potential=pot, use_voigt=use_voigt, stress_weight=0.5)
        calc.calculate(atoms, ["energy", "forces", "stress", "energies", "stresses"])
        r = calc.results
        assert abs(r["energies"].sum() - r["energy"]) <= 1e-6 * abs(r["energy"])
        assert np.abs(r["stresses"].astype(np.float64).sum(0) - r["stress"]).max() <= 1e-5 * np.abs(
            r["stress"]).max() + 1e-6
    # turning it off on the same model: the plain evaluation, no per-atom arrays
    plain = Potential_Dist(model=dm, element_refs=refs(model), **SCALING)
    E2, _F2, _S2, _ = plain(atoms)
    assert plain.atomic_energies is None and abs(float(E2) - float(E)) <= 1e-8 * abs(float(E))
    dm._engine.close()
