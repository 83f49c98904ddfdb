"""GPU: the balanced partition policy (b2m_set_partition_policy, DESIGN.md §4.1).

* the engine's walls equal tests/balance_ref.balanced_walls bit for bit (fed the graph_ref work of every atom), in a
  single-process group and in b2m_set_partition views, for a uniform, a two-phase, a particle (periodic and open) and a
  tilted cell, and for an unfolded heat-flux cell; where the restatement finds the width infeasible the engine fails
  with B2M_ERR_SLAB_WIDTH naming the same slab;
* the partition export with those walls equals GraphOracle's;
* a balanced group on one GPU computes what one partition computes (CHGNet, TensorNet, MACE small and medium);
* the default policy is untouched by a round trip through the balanced one.
"""
import functools

import numpy as np
import pytest

from distmlip_b200._lib import B2MError, PARTITION_BALANCED, PARTITION_EQUAL
from oracle import graph_ref as G
from tests import balance_ref as B
from tests._util import engine_from_model, engine_partition_digests, make_model, oracle_partition_digests
from tests.test_partition_balance import RB, RC, particle, tilted, two_phase, uniform

pytestmark = pytest.mark.gpu

STRUCTURES = {
    "uniform": lambda: uniform(3, 12, seed=3),
    "two_phase": lambda: two_phase(3, 12, seed=1),
    "particle": lambda: particle(24.0, seed=4),
    "particle_open": lambda: particle(24.0, seed=4, pbc=False),
    "tilted": lambda: tilted(),
}


@functools.lru_cache(maxsize=None)
def structure(name, rc=RC, rb=RB):
    atoms = STRUCTURES[name]()
    cart, lat, pbc = atoms.get_positions(), atoms.get_cell(), atoms.get_pbc().astype(np.int64)
    i1, _i2, _off, _d2, bond = G.neighbor_list(cart, lat, pbc, rc, rb)
    return atoms, B.engine_wrap(cart, lat, pbc), B.work_weights(i1, bond, len(cart))


def restated(name, P, rc=RC, rb=RB):
    """(axis, walls) or the SlabWidthError of the restatement, for a model with cutoffs rc and rb"""
    atoms, frac, w = structure(name, rc, rb)
    try:
        return B.balanced_partition(frac, atoms.get_cell(), atoms.get_pbc().astype(int), P, rc, rb, w)
    except B.SlabWidthError as e:
        return e


def set_structure(eng, atoms):
    eng.set_structure(atoms.get_positions(), atoms.get_cell(), np.zeros(len(atoms), dtype=np.int32),
                      atoms.get_pbc().astype(np.int32))


def check_walls(eng, atoms, ref, P):
    """every partition of `eng` (group views, or the one partition of a b2m_set_partition view) exports ref's walls"""
    if isinstance(ref, B.SlabWidthError):
        with pytest.raises(B2MError) as ei:
            set_structure(eng, atoms)
        assert ei.value.code == -4 and f"slab {ref.slab} " in str(ei.value), str(ei.value)
        return False
    set_structure(eng, atoms)
    for p in range(P if eng.group else 1):
        eng.set_view(p)
        assert eng.counts()["axis"] == ref[0]
        got = eng.partition_info(7)
        assert np.array_equal(got.view(np.int64), np.asarray(ref[1]).view(np.int64)), (p, got, ref[1])
    return True


@pytest.mark.parametrize("P", [2, 3, 4, 8])
@pytest.mark.parametrize("name", list(STRUCTURES))
def test_walls_bit_for_bit(name, P):
    atoms, _frac, _w = structure(name)
    ref = restated(name, P)
    model = make_model()
    group = engine_from_model(model, device=[0] * P)
    group.set_partition_policy(PARTITION_BALANCED)
    check_walls(group, atoms, ref, P)
    group.close()
    view = engine_from_model(model)
    view.set_partition_policy(PARTITION_BALANCED)
    for r in range(P):
        view.set_partition(r, P)
        check_walls(view, atoms, ref, P)
    view.close()


def test_unfolded_heat_flux_cell_walls():
    """the unfolded cell of the heat flux is partitioned without periodicity, walls measured from its lowest atom"""
    from oracle.heat_flux_ref import unfold

    atoms = two_phase(3, 6, seed=5)  # images within 10 A: shifts of -1, 0, 1 only, so positions are exact
    reach = 10.0
    ucart, _img = unfold(atoms.get_positions(), atoms.get_cell(), [1, 1, 1], reach)
    lat, open3 = atoms.get_cell(), np.zeros(3, dtype=np.int64)
    i1, _i2, _off, _d2, bond = G.neighbor_list(ucart, lat, open3, RC, RB)
    frac = B.engine_wrap(ucart, lat, open3)
    w = B.work_weights(i1, bond, len(ucart))
    for P in (2, 3):
        dim, walls = B.balanced_partition(frac, lat, open3, P, RC, RB, w, walls_from_min=True)
        eng = engine_from_model(make_model(), device=[0] * P)
        eng.set_partition_policy(PARTITION_BALANCED)
        eng.set_heat_flux(reach)
        set_structure(eng, atoms)
        for p in range(P):
            eng.set_view(p)
            assert eng.counts()["axis"] == dim
            assert np.array_equal(eng.partition_info(7).view(np.int64), walls.view(np.int64)), P
        eng.close()


@pytest.mark.parametrize("name,P", [("two_phase", 3), ("particle", 3), ("particle_open", 2), ("tilted", 2)])
def test_partition_export_matches_oracle(name, P):
    atoms, frac, _w = structure(name)
    dim, walls = restated(name, P)
    o = B.WalledOracle(atoms.get_positions(), atoms.get_cell(), atoms.get_pbc().astype(np.int64), dim, walls, RC, RB,
                       True, frac_wrapped=frac)
    eng = engine_from_model(make_model(), device=[0] * P)
    eng.set_partition_policy(PARTITION_BALANCED)
    set_structure(eng, atoms)
    for p in range(P):
        eng.set_view(p)
        assert engine_partition_digests(eng, P) == oracle_partition_digests(o, p), p
    eng.close()


def test_errors_and_policy_round_trip():
    atoms, _frac, _w = structure("two_phase")
    eng = engine_from_model(make_model(), device=[0, 0, 0])
    for bad in (-1, 2, 7):
        with pytest.raises(B2MError) as ei:
            eng.set_partition_policy(bad)
        assert ei.value.code == -1
    walls = []
    for policy in (PARTITION_EQUAL, PARTITION_BALANCED, PARTITION_EQUAL):
        eng.set_partition_policy(policy)
        set_structure(eng, atoms)
        walls.append(eng.partition_info(7).view(np.int64).copy())
    assert np.array_equal(walls[0], walls[2]) and not np.array_equal(walls[0], walls[1])
    ref = G.GraphOracle(atoms.get_positions(), atoms.get_cell(), np.array([1, 1, 1]), 3, RC, RB, True,
                        frac_wrapped=structure("two_phase")[1])
    assert np.array_equal(walls[0], ref.walls.view(np.int64))  # the reference's rule, bit for bit
    # infeasible: four 16 A slabs do not fit in the tilted cell's 46 A height; the slab is named
    t, _f, _w = structure("tilted")
    eng.set_partition_policy(PARTITION_BALANCED)
    with pytest.raises(B2MError) as ei:
        set_structure(eng, t)
    assert ei.value.code == -4 and "slab " in str(ei.value)
    set_structure(eng, atoms)  # the group stays usable
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# parity: a balanced group on one GPU against one partition
def _close(a, b, tol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())


def _chgnet(gpus, balance, atomic=False):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    dm = CHGNet_Dist.from_existing(make_model())
    dm.enable_distributed_mode(gpus, balance=balance)
    pot = Potential_Dist(model=dm, data_mean=0.5, data_std=1.5, calc_atomic=atomic)

    def run(atoms):
        E, F, S, _ = pot(atoms)
        out = [E.item(), F.numpy(), S.numpy()]
        if atomic:
            out += [pot.atomic_energies.numpy(), pot.atomic_stresses.numpy()]
        return out, dm._engine

    return run


def _tensornet(gpus, balance):
    from distmlip_b200.implementations.matgl import Potential_Dist, TensorNet_Dist
    from tests.test_oracle_tensornet import make_tn

    dm = TensorNet_Dist.from_existing(make_tn(seed=6, scale=1.5))
    dm.enable_distributed_mode(gpus, balance=balance)
    pot = Potential_Dist(model=dm)

    def run(atoms):
        E, F, S, _ = pot(atoms)
        return [E.item(), F.numpy(), S.numpy()], dm._engine

    return run


def _mace(gpus, balance, medium):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist
    from oracle.mace_ref import make_mace
    from tests.mace_eq_ref import make_mace_eq

    m = (make_mace_eq if medium else make_mace)(seed=4, C=32, r_max=5.0, scale=8.0)
    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode(gpus, balance=balance)

    def run(atoms):
        e, f, s, ae, av = d.evaluate(atoms, atomic=True)
        return [e, f, s, ae, av], d._engine

    return run


# builder, energy and force / stress tolerances (those of test_gpu_group.py and the MACE group tests), cutoffs
FAMILIES = {
    "chgnet": (_chgnet, 1e-7, 2e-6, (RC, RB)),
    "tensornet": (_tensornet, 1e-6, 1e-5, (5.0, 0.0)),
    "mace_small": (lambda g, b: _mace(g, b, False), 1e-6, 1e-5, (5.0, 0.0)),
    "mace_medium": (lambda g, b: _mace(g, b, True), 1e-6, 1e-5, (5.0, 0.0)),
}


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("name", ["two_phase", "particle"])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_balanced_group_equals_one_partition(family, name, P):
    make, tol_e, tol_f, cutoffs = FAMILIES[family]
    atoms, _frac, _w = structure(name)
    one, eng1 = make([0], False)(atoms)
    many, eng = make([0] * P, True)(atoms)
    n = len(atoms)
    assert abs(one[0] - many[0]) / n < tol_e * max(1.0, abs(one[0]) / n)
    for a, b in zip(many[1:], one[1:]):
        assert _close(a, b, tol_f)
    c = eng.counts()
    assert c["world"] == P and c["n_halo"] > 0
    ref = restated(name, P, *cutoffs)  # without a bond graph the work is the edges alone
    assert np.array_equal(eng.partition_info(7).view(np.int64), ref[1].view(np.int64))
    eng.close(), eng1.close()


def test_balanced_group_per_atom_chgnet():
    atoms, _frac, _w = structure("two_phase")
    one, e1 = _chgnet([0], False, atomic=True)(atoms)
    many, e3 = _chgnet([0, 0, 0], True, atomic=True)(atoms)
    assert _close(many[3], one[3], 1e-6) and _close(many[4], one[4], 2e-5)
    assert abs(many[3].sum() - many[0]) < 1e-6 * max(1.0, abs(many[0]))
    e1.close(), e3.close()


def test_balanced_group_heat_flux_chgnet():
    atoms = two_phase(3, 6, seed=5)
    v = np.random.default_rng(3).normal(0.0, 0.01, size=(len(atoms), 3))
    out = []
    for devs, policy in (([0], PARTITION_EQUAL), ([0, 0], PARTITION_BALANCED)):
        eng = engine_from_model(make_model(), device=devs)
        eng.set_partition_policy(policy)
        eng.set_heat_flux(10.0)
        set_structure(eng, atoms)
        out.append(eng.compute_heat_flux(v))
        eng.close()
    (e1, f1, s1, (jp1, jc1)), (e2, f2, s2, (jp2, jc2)) = out
    assert abs(e1 - e2) / len(atoms) < 1e-7 * max(1.0, abs(e1) / len(atoms))
    assert _close(f2, f1, 2e-6) and _close(s2, s1, 2e-6)
    assert _close(jp2, jp1, 1e-5) and _close(jc2, jc1, 1e-5)
