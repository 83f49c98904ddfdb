"""MACE with hidden features C x 0e + C x 1o + C x 2e (the MACE-MP-0 "large" shape) on the H100 engine against the f64
oracle (tests/mace_l2_ref.py), with the thresholds of test_gpu_mace_equivariant.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from tests.mace_eq_ref import make_mace_eq
from tests.mace_l2_ref import (RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock, atomic_virials_ref,
                               make_mace_l2, make_mace_l2_core, potential_ref)

pytestmark = pytest.mark.gpu

SYMS = ("Si", "C", "O")


def mixed(atoms, seed=0):
    rng = np.random.default_rng(seed)
    sy = [SYMS[k] for k in rng.integers(0, len(SYMS), len(atoms))]
    return SimpleAtoms(sy, atoms.get_positions(), np.array(atoms.get_cell()), pbc=atoms.get_pbc())


def model(**kw):
    kw.setdefault("C", 32)
    kw.setdefault("r_max", 6.0)
    kw.setdefault("scale", 8.0)
    return make_mace_l2(**kw)


def run(m, atoms, gpus=(0,)):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode(list(gpus))
    return d, d.evaluate(atoms, atomic=True)


def check(m, atoms, gpus=(0,)):
    E, F, S, eps = potential_ref(m, atoms)
    d, (e, f, s, ae, av) = run(m, atoms, gpus)
    d._engine.close()
    n = len(atoms)
    de = abs(e - E.item()) / n
    df = np.abs(f - F.numpy()).max()
    ds = np.abs(s - S.numpy()).max()
    print(f"n={n} dE/atom={de:.2e} dF={df:.2e} dS={ds:.2e} |F|max={F.abs().max():.3f}")
    assert de < 1e-4 and df < 1e-3 and ds < 1e-3, (de, df, ds)
    assert np.abs(ae - eps.numpy()).max() < 1e-4
    return e, f, s, ae, av


@pytest.mark.parametrize("correlation", [1, 2, 3])
@pytest.mark.parametrize("max_ell", [2, 3])
def test_diamond_mixed(correlation, max_ell):
    check(model(correlation=correlation, max_ell=max_ell, seed=correlation + 10 * max_ell),
          mixed(si_diamond(2, seed=1)))  # 64 atoms


def test_c128_max_ell_3():
    check(model(C=128, seed=21), mixed(si_diamond(2, seed=2)))


def test_three_layers_residual_only():
    """layer 1 takes and gives 0e+1o+2e: the three-block residual skip"""
    cls = [RealAgnosticResidualInteractionBlock] * 3
    check(model(num_interactions=3, interaction_classes=cls, seed=4), mixed(si_diamond(2, seed=4)))


def test_three_layers_plain_classes_c96_max_ell_2():
    cls = [RealAgnosticInteractionBlock, RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock]
    check(model(C=96, num_interactions=3, interaction_classes=cls, max_ell=2, seed=5), mixed(si_diamond(2, seed=3)))


def test_rough_cell():
    check(model(seed=6), mixed(rough_cell(200, seed=1), seed=2))


def test_cluster_non_periodic():
    a = si_diamond(2, seed=4)
    c = SimpleAtoms(["Si"] * len(a), a.get_positions(), np.eye(3) * 40.0, pbc=(False, False, False))
    check(model(seed=7), mixed(c, seed=3))


def test_large_cell_loops():
    # 4096 atoms: every per-atom grid covers the 132 SMs several times; r_max 4 A keeps the float64 oracle's autograd
    # graph (17 paths per edge) within host memory
    check(model(seed=8, r_max=4.0), mixed(si_diamond(8, seed=5)))


@pytest.mark.parametrize("parts", [2, 3])
def test_group_partitions_equal_one(parts):
    m = model(seed=9, num_interactions=3)
    atoms = mixed(si_diamond(3, nz=10, seed=6))
    _, (e1, f1, s1, a1, v1) = run(m, atoms)
    _, (e2, f2, s2, a2, v2) = run(m, atoms, gpus=[0] * parts)
    assert abs(e1 - e2) / len(atoms) < 1e-6
    assert np.abs(f1 - f2).max() < 1e-5 and np.abs(s1 - s2).max() < 1e-5
    assert np.abs(a1 - a2).max() < 1e-5 and np.abs(v1 - v2).max() < 1e-5


def test_atomic_virials_and_sum_rules():
    m = model(seed=10)
    atoms = mixed(si_diamond(2, seed=7))
    e, f, s, ae, av = check(m, atoms)
    w = atomic_virials_ref(m, atoms).numpy()
    assert np.abs(av - w).max() < 1e-4 * max(1.0, np.abs(w).max()), np.abs(av - w).max()
    assert abs(ae.sum() - e) < 1e-6 * max(1.0, abs(e))
    vol = atoms.get_volume()
    np.testing.assert_allclose(av.sum(axis=0), s * vol / 160.21766208, atol=2e-4)


def test_h1_stage_tap():
    """h1 ([n_own][9][C]: 0e, 1o m = 0..2, 2e m = 0..4) against the oracle's tap"""
    m = model(C=64, seed=11)
    atoms = mixed(si_diamond(2, seed=8))
    taps = {}
    potential_ref(m, atoms, calc_forces=False, taps=taps)
    d, _ = run(m, atoms)
    h1 = d._engine.debug_tensor("h1")
    assert h1.shape == (len(atoms), 9 * 64)
    ref = taps["h1"].numpy().reshape(len(atoms), 9 * 64)
    assert np.abs(h1 - ref).max() < 1e-4 * max(1.0, np.abs(ref).max()), np.abs(h1 - ref).max()
    assert np.abs(ref[:, 4 * 64:]).max() > 1e-3  # the 2e part is not trivially zero


def test_zbl_agnesi_on_large_shape():
    m = make_mace_l2_core(seed=15, C=32, r_max=6.0, scale=8.0)
    assert m.pair_repulsion
    check(m, mixed(si_diamond(2, seed=10)))


def test_heat_flux_small_cell():
    from tests import mace_heat_flux_ref as HF

    m = model(seed=16, r_max=4.0)
    atoms = mixed(si_diamond(1, seed=11))
    v = np.random.default_rng(3).normal(size=(len(atoms), 3))
    d, _ = run(m, atoms)
    e, f, s, ae, av, (jp, jc) = d.evaluate_heat_flux(atoms, v, atomic=True)
    ref = HF.heat_flux_ref(m, atoms, v)
    jp_ref, jc_ref = np.asarray(ref["j_pot"]), np.asarray(ref["j_conv"])
    assert abs(e - ref["energy"]) / len(atoms) < 1e-4
    scale = max(1.0, np.abs(jp_ref).max())
    assert np.abs(jp - jp_ref).max() < 1e-4 * scale, (jp, jp_ref)
    assert np.abs(jc - jc_ref).max() < 1e-4 * max(1.0, np.abs(jc_ref).max()), (jc, jc_ref)


def test_calculator_committee_medium_and_large():
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    class Calc:  # the attribute surface of mace's MACECalculator
        def __init__(self, models):
            self.models, self.r_max = models, 6.0
            self.energy_units_to_eV, self.length_units_to_A = 1.0, 1.0

    ms = [make_mace_eq(seed=12, C=32, r_max=6.0, scale=8.0), model(seed=13)]
    atoms = mixed(si_diamond(2, seed=9))
    n = len(atoms)
    calc = MACECalculator_Dist.from_existing(Calc(ms))
    calc.enable_distributed_mode([0])
    calc.calculate(atoms)
    r = calc.results
    refs = [potential_ref(m, atoms) for m in ms]
    E = np.array([x[0].item() for x in refs])
    F = np.stack([x[1].numpy() for x in refs])
    assert abs(r["energy"] - E.mean()) / n < 1e-4
    np.testing.assert_allclose(r["energies"], E, atol=1e-4 * n)
    np.testing.assert_allclose(r["forces_comm"], F, atol=1e-3)
    np.testing.assert_allclose(r["forces"], F.mean(0), atol=1e-3)


def test_engine_rejects_2e_with_max_ell_1():
    from distmlip_b200 import _lib
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    desc = ScaleShiftMACE_Dist.from_existing(model(seed=14))._describe()
    desc.max_ell = 1
    with pytest.raises(Exception, match="max_ell"):
        _lib.Engine(n_elem=desc.n_elem, n_blocks=desc.num_interactions, cutoff=desc.r_max, mace=desc, device=0)
