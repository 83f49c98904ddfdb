"""The batched relaxation's restatement (tests/relax_ref.py) on the CPU: the Frechet cell force is the gradient of
-(E + pV) in X, FIRE + the filter relaxes a Lennard-Jones fcc crystal to its analytic lattice constant (p = 0) and
volume (p > 0), and, where a real ASE is installed, it matches ASE's FIRE + FrechetCellFilter step for step."""
import numpy as np
import pytest
from scipy.linalg import expm
from scipy.optimize import minimize_scalar

from tests.relax_ref import FIRE_DEFAULTS, Fire, cell_force, fcc, lj, relax


def strained_cell(seed=0):
    rng = np.random.default_rng(seed)
    pos, cell = fcc(3.1, reps=2)
    strain = np.eye(3) + 0.04 * rng.standard_normal((3, 3))
    return pos @ strain.T + 0.05 * rng.standard_normal(pos.shape), cell @ strain.T


@pytest.mark.parametrize("p", [0.0, 0.003])
def test_cell_force_is_minus_the_gradient_in_x(p):
    pos0, cell0 = strained_cell(1)
    n = len(pos0)
    X = 0.3 * np.random.default_rng(2).standard_normal((3, 3))  # a non-trivial, non-symmetric current deformation

    def H(Xv):
        F = expm(Xv / n)
        cell = cell0 @ F.T
        E, _, _ = lj(pos0 @ F.T, cell)
        return E + p * abs(np.linalg.det(cell))

    F = expm(X / n)
    cell = cell0 @ F.T
    _, f, W = lj(pos0 @ F.T, cell)
    got = cell_force(X, W, abs(np.linalg.det(cell)), n, k=1.0, p=p)
    h = 1e-4
    want = np.zeros((3, 3))
    for a in range(3):
        for b in range(3):
            d = np.zeros((3, 3))
            d[a, b] = h
            want[a, b] = -(H(X + d) - H(X - d)) / (2 * h)
    np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-7 * np.abs(want).max())
    # and the atom rows: f F = -dE/dr0
    opt = Fire(pos0, cell0, True, p=p)
    opt.X = X
    g = opt.forces(f, W)[:n]
    i = 3
    fd = np.zeros(3)
    for a in range(3):
        r = pos0.copy()
        r[i, a] += h
        ep = lj(r @ F.T, cell)[0]
        r[i, a] -= 2 * h
        em = lj(r @ F.T, cell)[0]
        fd[a] = -(ep - em) / (2 * h)
    np.testing.assert_allclose(g[i], fd, rtol=1e-7, atol=1e-9)


def lattice_minimum(p):
    """the fcc lattice constant minimising E + pV of the LJ crystal (a 1-D minimisation of the lattice sum)"""
    def H(a):
        pos, cell = fcc(a, reps=2)
        return lj(pos, cell)[0] + p * a ** 3 * 8

    return minimize_scalar(H, bounds=(2.6, 3.6), method="bounded", options=dict(xatol=1e-10)).x


@pytest.mark.parametrize("p", [0.0, 0.002])
def test_lj_fcc_relaxes_to_the_analytic_volume(p):
    a_star = lattice_minimum(p)
    pos, cell = strained_cell(3)
    out = relax([(pos, cell)], lambda ids, geos: [lj(x, c) for x, c in geos], fmax=1e-5, steps=3000,
                relax_cell=True, p=p)[0]
    assert out["converged"], out["steps"]
    V = abs(np.linalg.det(out["cell"]))
    np.testing.assert_allclose(V, 8 * a_star ** 3, rtol=1e-5)
    # the relaxed cell is fcc: its metric is a multiple of a rotated cube's
    G = out["cell"] @ out["cell"].T
    np.testing.assert_allclose(np.sort(np.linalg.eigvalsh(G)), (2 * a_star) ** 2 * np.ones(3), rtol=1e-4)


def test_structures_do_not_couple_and_stop_at_steps():
    a = strained_cell(4)
    b = strained_cell(5)
    ev = lambda ids, geos: [lj(x, c) for x, c in geos]  # noqa: E731
    both = relax([a, b], ev, fmax=0.0, steps=7, relax_cell=True)
    alone = relax([b], ev, fmax=0.0, steps=7, relax_cell=True)[0]
    assert both[1]["steps"] == 7 and not both[1]["converged"] and len(both[1]["energies"]) == 8
    np.testing.assert_array_equal(both[1]["positions"], alone["positions"])
    np.testing.assert_array_equal(both[1]["cell"], alone["cell"])


def _real_ase():
    try:
        import ase
        from ase.filters import FrechetCellFilter  # noqa: F401
        from ase.optimize import FIRE  # noqa: F401
    except Exception:  # noqa: BLE001
        return None
    return None if getattr(ase, "IS_STUB", False) else ase


@pytest.mark.parametrize("relax_cell", [False, True])
def test_matches_ase_step_for_step(relax_cell):
    ase = _real_ase()
    if ase is None:
        pytest.skip("ASE with FIRE and FrechetCellFilter is not installed")
    from ase.calculators.calculator import Calculator, all_changes
    from ase.filters import FrechetCellFilter
    from ase.optimize import FIRE

    class LJ(Calculator):
        implemented_properties = ["energy", "forces", "stress"]

        def calculate(self, atoms=None, properties=None, system_changes=all_changes):
            super().calculate(atoms, properties, system_changes)
            E, f, W = lj(atoms.positions, np.array(atoms.cell))
            s = W / atoms.get_volume()
            self.results = dict(energy=E, forces=f, stress=np.array([s[0, 0], s[1, 1], s[2, 2], s[1, 2], s[0, 2],
                                                                       s[0, 1]]))

    pos, cell = strained_cell(6)
    atoms = ase.Atoms("Ar" * len(pos), positions=pos, cell=cell, pbc=True)
    atoms.calc = LJ()
    traj = []
    target = FrechetCellFilter(atoms, scalar_pressure=0.001) if relax_cell else atoms
    opt = FIRE(target, logfile=None)
    opt.attach(lambda: traj.append((atoms.positions.copy(), np.array(atoms.cell))))
    opt.run(fmax=0.0, steps=12)
    out = relax([(pos, cell)], lambda ids, geos: [lj(x, c) for x, c in geos], fmax=0.0, steps=12,
                relax_cell=relax_cell, p=0.001 if relax_cell else 0.0)[0]
    assert len(traj) == len(out["geometries"]) == 13
    for (xa, ca), (xr, cr) in zip(traj, out["geometries"]):
        np.testing.assert_allclose(xr, xa, atol=1e-9)
        np.testing.assert_allclose(cr, ca, atol=1e-9)


def test_fire_defaults_are_the_librarys():
    from distmlip_b200 import _lib

    assert _lib.FIRE_DEFAULTS == FIRE_DEFAULTS
