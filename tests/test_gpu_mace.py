"""MACE (ScaleShiftMACE, hidden_irreps = C x 0e) on the H100 engine against the f64 oracle (oracle/mace_ref.py)."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.mace_ref import (RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock, atomic_virials_ref,
                             make_mace, potential_ref)

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
    return make_mace(**kw)


def run(m, atoms, gpus=(0,)):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode(list(gpus))
    return d, d.evaluate(atoms, atomic=True)


def check(m, atoms, gpus=(0,)):
    E, F, S, eps = potential_ref(m, atoms)
    _, (e, f, s, ae, av) = run(m, atoms, gpus)
    n = len(atoms)
    de = abs(e - E.item()) / n
    df = np.abs(f - F.numpy()).max()
    ds = np.abs(s - S.numpy()).max()
    print(f"n={n} dE/atom={de:.2e} dF={df:.2e} dS={ds:.2e} |F|max={F.abs().max():.3f}")
    assert de < 1e-4 and df < 1e-3 and ds < 1e-3, (de, df, ds)
    assert np.abs(ae - eps.numpy()).max() < 1e-4
    return e, f, s, ae, av


@pytest.mark.parametrize("correlation", [1, 2, 3])
def test_diamond_mixed(correlation):
    check(model(correlation=correlation, seed=correlation), mixed(si_diamond(2, seed=1)))  # 64 atoms


def test_diamond_512_c128_residual_only():
    cls = [RealAgnosticResidualInteractionBlock] * 2
    check(model(C=128, interaction_classes=cls, seed=4), mixed(si_diamond(4, seed=2)))


def test_nonresidual_layers_and_c96():
    cls = [RealAgnosticInteractionBlock, RealAgnosticInteractionBlock, RealAgnosticResidualInteractionBlock]
    check(model(C=96, num_interactions=3, interaction_classes=cls, max_ell=2, seed=5), mixed(si_diamond(2, seed=3)))


def test_rough_cell_c64():
    check(model(C=64, seed=6), mixed(rough_cell(200, seed=1), seed=2))


def test_64_bessel_functions():
    # w_n d reaches 64 pi: the radial basis and its derivative far outside [-pi, pi]
    check(model(num_bessel=64, seed=13), mixed(si_diamond(2, seed=9)))


def test_inert_e3nn_buffers():
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    m = model(seed=14)
    atoms = mixed(si_diamond(2, seed=10))
    d = ScaleShiftMACE_Dist.from_existing(m)
    d._state_dict["interactions.0.linear_up.output_mask"] = torch.ones(32)
    d._state_dict["interactions.0.conv_tp.weight"] = torch.zeros(0)
    d.enable_distributed_mode([0])
    e = d.evaluate(atoms)[0]
    assert abs(e - potential_ref(m, atoms, calc_forces=False)[0].item()) / len(atoms) < 1e-4
    d = ScaleShiftMACE_Dist.from_existing(m)
    mask = torch.ones(32)
    mask[3] = 0.0
    d._state_dict["interactions.1.linear.output_mask"] = mask
    with pytest.raises(Exception, match="output_mask"):
        d.enable_distributed_mode([0])


def test_cluster_non_periodic():
    a = si_diamond(2, seed=4)
    c = SimpleAtoms(["Si"] * len(a), a.get_positions(), np.eye(3) * 40.0, pbc=(False, False, False))
    check(model(seed=7), mixed(c, seed=3))


def test_large_cell_loops():
    # 4096 atoms, ~ 0.3 M edges: every per-atom grid covers the 132 SMs several times, the edge GEMMs ~ 2 000 tiles
    check(model(seed=8), mixed(si_diamond(8, seed=5)))


@pytest.mark.parametrize("parts", [2, 3])
def test_group_partitions_equal_one(parts):
    m = model(seed=9)
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


def test_calculator_committee_md():
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    class Calc:  # the attribute surface of mace's MACECalculator
        def __init__(self, models, eu=1.0):
            self.models, self.r_max = models, 6.0
            self.energy_units_to_eV, self.length_units_to_A = eu, 1.0

    ms = [model(seed=11), model(seed=12)]
    atoms = mixed(si_diamond(2, seed=8))
    n = len(atoms)
    calc = MACECalculator_Dist.from_existing(Calc(ms))
    calc.enable_distributed_mode([0])
    calc.calculate(atoms)
    r = calc.results
    refs = [potential_ref(m, atoms) for m in ms]
    E = np.array([x[0].item() for x in refs])
    F = np.stack([x[1].numpy() for x in refs])
    S = np.stack([x[2].numpy() / 160.21766208 for x in refs])  # eV / A^3
    voigt = lambda t: np.array([t[0, 0], t[1, 1], t[2, 2], t[1, 2], t[0, 2], t[0, 1]])  # noqa: E731
    assert abs(r["energy"] - E.mean()) / n < 1e-4 and r["free_energy"] == r["energy"]
    np.testing.assert_allclose(r["energies"], E, atol=1e-4 * n)
    assert abs(r["energy_var"] - E.var()) < 1e-3 * max(1.0, E.var())
    np.testing.assert_allclose(r["forces"], F.mean(0), atol=1e-3)
    np.testing.assert_allclose(r["forces_comm"], F, atol=1e-3)
    np.testing.assert_allclose(r["stress"], voigt(S.mean(0)), atol=1e-5)
    np.testing.assert_allclose(r["stress_var"], voigt(S.var(0)), atol=1e-8)
    e0 = ms[0].atomic_energies_fn.atomic_energies.numpy()
    z_index = [ms[0].atomic_numbers.tolist().index(z) for z in atoms.get_atomic_numbers()]
    node = np.mean([x[3].numpy() for x in refs], axis=0) - e0[z_index]
    np.testing.assert_allclose(r["node_energy"], node, atol=1e-4)
    # energy units: everything in eV scales with energy_units_to_eV
    calc2 = MACECalculator_Dist.from_existing(Calc([ms[0]], eu=2.0))
    calc2.enable_distributed_mode([0])
    calc2.calculate(atoms)
    assert abs(calc2.results["energy"] - 2.0 * E[0]) / n < 2e-4
    np.testing.assert_allclose(calc2.results["forces"], 2.0 * F[0], atol=2e-3)
    np.testing.assert_allclose(calc2.results["stress"], 2.0 * voigt(S[0]), atol=2e-5)
    # three velocity-Verlet steps with the calculator's forces; the last state against the oracle
    pos = atoms.get_positions().copy()
    vel = np.zeros_like(pos)
    mass, dt = 28.0, 1.0
    for _ in range(3):
        vel += 0.5 * dt * calc.results["forces"] / mass
        pos += dt * vel
        moved = SimpleAtoms(atoms.get_chemical_symbols(), pos, np.array(atoms.get_cell()))
        calc.calculate(moved)
        vel += 0.5 * dt * calc.results["forces"] / mass
    assert np.abs(pos - atoms.get_positions()).max() > 1e-4
    refs = [potential_ref(m, moved) for m in ms]
    assert abs(calc.results["energy"] - np.mean([x[0].item() for x in refs])) / n < 1e-4
    np.testing.assert_allclose(calc.results["forces"], np.mean([x[1].numpy() for x in refs], axis=0), atol=1e-3)
