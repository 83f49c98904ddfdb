"""GPU: per-atom energies and per-atom virials (b2m_set_atomic / b2m_get_atomic) of CHGNet and TensorNet against the
autograd oracle (oracle/atomic_ref.py), their sum rules against the engine's own energy and stress, partition
independence in single-process groups, the off -> on -> off round trip on one handle, and PESCalculator_Dist.

The tolerances are fp32 round-off, not accuracy targets.  A kernel that adds an edge's half to the wrong atom keeps both
sum rules, so only the per-atom comparison sees it; tests/test_atomic_oracle.py checks that these tolerances stay at
least 10x below the error of such routing bugs and below a tenth of a single edge's contribution.  The per-atom
virials are compared relative to max |w_ref| of the structure; the per-atom energies absolutely."""
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
# Observed on an H100 over every comparison in this file: max |d eps| 2.4e-7 eV, max |dw| / max |w| 4.1e-6 (CHGNet) and
# 2.0e-6 (TensorNet)
TOL_EPS = 2e-6                                 # eV, max |eps - eps_ref| over the atoms
TOL_W = {"chgnet": 4e-5, "tensornet": 2e-5}    # max |w - w_ref| over atoms and components, over max |w_ref|
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


def oracle(family, atoms, edges=False):
    model = model_of(family)
    return atomic_ref(model, atoms, element_refs=refs(model), dtype=torch.float64, edges=edges, **SCALING)


def check_against_oracle(family, eps, w, ref, what=""):
    wref = ref["virials"].numpy()
    de = np.abs(eps - ref["energies"].numpy()).max()
    dw = np.abs(w - wref).max() / np.abs(wref).max()
    print(f"per-atom error {family} {what}: max|d eps| {de:.2e} eV, max|dw| / max|w| {dw:.2e} "
          f"(max|w| {np.abs(wref).max():.2e} eV)")
    assert de <= TOL_EPS, de
    assert dw <= TOL_W[family], dw


def check_same_per_atom_values(family, eps, w, eps0, w0, tol_eps, tol_w, what=""):
    """two engine evaluations of the same atoms (fp32 sums in a different order)"""
    de = np.abs(eps - eps0).max()
    dw = np.abs(w - w0).max() / np.abs(w0).max()
    print(f"per-atom difference {family} {what}: max|d eps| {de:.2e} eV, max|dw| / max|w| {dw:.2e}")
    assert de <= tol_eps, de
    assert dw <= tol_w, dw


def check_sum_rules(eps, w, e, s, volume):
    assert abs(eps.sum() - e) <= 1e-6 * abs(e), (eps.sum(), e)
    sig = w.astype(np.float64).sum(0) / volume * GPA_PER_EVA3
    assert np.abs(sig - s).max() <= 1e-5 * np.abs(s).max() + 1e-6, (sig, s)


STRUCTURES = {
    "diamond64": lambda: mixed(si_diamond(2, sigma=0.15, seed=1)),
    "diamond512": lambda: mixed(si_diamond(4, sigma=0.15, seed=2)),
    "rough": lambda: mixed(rough_cell(300, seed=4), other="Ge", every=2),
}


def slab():
    """three 21.7 A slabs: the partition test's cell"""
    return mixed(si_diamond(2, sigma=0.15, seed=5, nz=12))


def calculator_cell():
    """the calculator test's cell"""
    return mixed(si_diamond(2, sigma=0.15, seed=8, nz=8))


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
    check_against_oracle(family, eps, w, oracle(family, atoms), structure)
    check_sum_rules(eps, w, e, s, atoms.get_volume())
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_partitions_of_a_group_give_the_same_per_atom_values(family):
    atoms = slab()
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
        check_against_oracle(family, eps, w, ref, f"slab, {len(devs)} partitions")
        check_sum_rules(eps, w, e, s, atoms.get_volume())
        got.append((eps, w))
        eng.close()
    for k, (eps, w) in enumerate(got[1:], 2):  # fp32 atomics in a different order: round-off level
        check_same_per_atom_values(family, eps, w, *got[0], TOL_EPS, TOL_W[family], f"slab, {k} vs 1 partitions")


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
    assert np.abs(eps2 - eps).max() <= TOL_EPS
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

    atoms = calculator_cell()
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
    check_against_oracle(family, pot.atomic_energies.numpy(),
                         pot.atomic_stresses.numpy().astype(np.float64) * atoms.get_volume() / GPA_PER_EVA3, ref,
                         f"calculator, {len(devices)} partitions")
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


# ------------------------------------------------------------------ where the destination-run reduction can misroute
def rough4000():
    """4000 atoms, about 100 k edges, in-degree up to 35: the engine's edge order has destination runs longer than a
    warp, runs cut by warp boundaries and runs that end on lane 31"""
    return mixed(rough_cell(4000, seed=11), other="Ge", every=2)


def irregular():
    """random cell stretched along the slab axis (68 A along z): uneven partitions and halo sections"""
    return mixed(rough_cell(1000, seed=12, aspect=(1, 1, 4)), other="Ge", every=2)


def dst_runs(dst):
    """first and last position of every run of equal destinations in an edge list"""
    start = np.r_[True, dst[1:] != dst[:-1]]
    first = np.flatnonzero(start)
    return first, np.r_[first[1:] - 1, len(dst) - 1]


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_per_atom_values_match_the_oracle_at_4000_atoms(family):
    from oracle.atomic_ref import routing_mutants
    from tests._util import key5

    atoms = rough4000()
    model = model_of(family)
    eng = engine_of(family, model)
    set_structure(eng, model, atoms)
    eng.set_atomic(True)
    e, _f, s = eng.compute(forces=True, stress=True)
    eps, w = eng.atomic()
    edges = eng.partition_info(3)  # (src, dst, image) in the order of the per-edge kernels: lane = edge % 32
    first, last = dst_runs(edges[:, 1])
    print(f"{len(edges)} edges, longest run {int((last - first).max()) + 1}, "
          f"{int((first // 32 != last // 32).sum())} runs cut by a warp boundary, {int((last % 32 == 31).sum())} end on "
          f"lane 31")
    assert (last - first + 1).max() > 32
    assert (first // 32 != last // 32).sum() > 100
    assert (last[:-1] % 32 == 31).any()
    ref = oracle(family, atoms, edges=True)
    check_against_oracle(family, eps, w, ref, "rough4000")
    check_sum_rules(eps, w, e, s, atoms.get_volume())
    # the routing bugs of the engine's own edge order stay 10x above the tolerance on this structure
    okey = {k: i for i, k in enumerate(key5(np.column_stack([ref["edge_src"], ref["edge_dst"], ref["edge_off"]])))}
    order = np.array([okey[k] for k in key5(edges)], dtype=np.int64)
    wref = ref["virials"]
    for name, wm in routing_mutants(ref["edge_src"], ref["edge_dst"], ref["edge_half"], len(atoms), order).items():
        if family == "chgnet" and name == "src_transposed":
            continue  # CHGNet's per-atom virials are symmetric to 1e-4 of max |w|: a transposition is invisible
        err = float((wm - wref).abs().max())
        assert err >= 10 * TOL_W[family] * float(wref.abs().max()), (name, err)
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("parts", [2, 3])
def test_groups_on_an_irregular_cell(family, parts):
    """CHGNet's bonds that cross a partition boundary are split by k_halo_bond_final<kAtomic>; the leader sums the
    partitions' arrays"""
    atoms = irregular()
    model = model_of(family)
    eng = engine_of(family, model, device=[0] * parts)
    set_structure(eng, model, atoms)
    eng.set_atomic(True)
    e, _f, s = eng.compute(forces=True, stress=True)
    c = [eng.counts(partition=p) for p in range(parts)]
    assert c[0]["world"] == parts
    print("partitions (owned, halo, halo bonds):", [(x["n_own"], x["n_halo"], x["n_bond_halo"]) for x in c])
    if family == "chgnet":
        assert all(x["n_bond_halo"] > 0 for x in c)
    eps, w = eng.atomic()
    check_against_oracle(family, eps, w, oracle(family, atoms), f"rough 1x1x4, {parts} partitions")
    check_sum_rules(eps, w, e, s, atoms.get_volume())
    eng.close()


# ------------------------------------------------------------- metamorphic, at sizes the oracle cannot reach
# the same atoms evaluated twice: the graph, the edge order and the fp32 sums differ, nothing else.  Tolerances:
# per-atom energies absolute (eV), per-atom virials over max |w|; observed on an H100: 8.9e-8 eV and 1.1e-6.
TOL_SAME_EPS = 5e-7
TOL_SAME_W = 1e-5
BIG = {"chgnet": lambda: mixed(si_diamond(23, sigma=0.15, seed=13)),        # 97 336 atoms (bench.py --cells 23)
       "tensornet": lambda: mixed(si_diamond(12, sigma=0.15, seed=13))}    # 13 824 atoms


def atomic_of(eng, model, atoms):
    set_structure(eng, model, atoms)
    eng.compute(forces=True, stress=True)
    return eng.atomic()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_permuting_the_atoms_permutes_the_per_atom_values(family):
    """a new atom order moves every atom to other CSR positions, other runs and other warps"""
    atoms = BIG[family]()
    model = model_of(family)
    eng = engine_of(family, model)
    eng.set_atomic(True)
    eps, w = atomic_of(eng, model, atoms)
    perm = np.random.default_rng(14).permutation(len(atoms))
    sym = np.array(atoms.get_chemical_symbols())[perm].tolist()
    eps_p, w_p = atomic_of(eng, model, SimpleAtoms(sym, atoms.get_positions()[perm], atoms.get_cell()))
    check_same_per_atom_values(family, eps_p, w_p, eps[perm], w[perm], TOL_SAME_EPS, TOL_SAME_W,
                               f"{len(atoms)} atoms, permuted")
    eng.close()


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
def test_repeating_the_cell_repeats_the_per_atom_values(family):
    """the cell twice along z: every atom and its image have the same neighbourhood, hence the same values, except
    for the data_mean / N share of each per-atom energy"""
    atoms = BIG[family]()
    model = model_of(family)
    eng = engine_of(family, model)
    eng.set_atomic(True)
    eps, w = atomic_of(eng, model, atoms)
    cell = np.array(atoms.get_cell())
    pos = atoms.get_positions()
    twice = SimpleAtoms(atoms.get_chemical_symbols() * 2, np.concatenate([pos, pos + cell[2]]),
                        cell * np.array([[1.0], [1.0], [2.0]]))
    eps2, w2 = atomic_of(eng, model, twice)
    n = len(atoms)
    eps2 = eps2 - SCALING["data_mean"] / (2 * n) + SCALING["data_mean"] / n
    for k in range(2):
        check_same_per_atom_values(family, eps2[k * n:(k + 1) * n], w2[k * n:(k + 1) * n], eps, w, TOL_SAME_EPS,
                                   TOL_SAME_W, f"{n} atoms, image {k} of the doubled cell")
    eng.close()
