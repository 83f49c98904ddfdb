"""CPU: the per-atom energy / virial oracle (oracle/atomic_ref.py) for CHGNet and TensorNet, and the ASE calculator's
`energies` / `stresses` with a Potential_Dist double.

The oracle's sum rules are identities: per-atom energies sum to the energy, the edge-split per-atom virials sum to the
strain derivative that `stress` is made of.  Both hold to f64 round-off.
"""
import os
import sys

import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.atomic_ref import atomic_ref
from tests._util import make_model
from tests.test_oracle_tensornet import make_tn

HERE = os.path.dirname(os.path.abspath(__file__))
GPA_PER_EVA3 = 160.21766208


def mixed(atoms, other="O", every=3):
    sym = [other if i % every == 0 else s for i, s in enumerate(atoms.get_chemical_symbols())]
    return SimpleAtoms(sym, atoms.get_positions(), atoms.get_cell())


def model_of(family):
    return make_model(seed=2) if family == "chgnet" else make_tn(seed=3, scale=1.5)


STRUCTURES = {
    "diamond": lambda: mixed(si_diamond(2, sigma=0.15, seed=1)),
    "rough": lambda: mixed(rough_cell(48, seed=4), other="Ge", every=2),
}
SCALING = dict(data_mean=0.7, data_std=1.3)


def refs(model):
    return np.linspace(-0.5, 0.5, len(model.element_types))


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("structure", list(STRUCTURES))
def test_sum_rules(family, structure):
    atoms = STRUCTURES[structure]()
    model = model_of(family)
    r = atomic_ref(model, atoms, element_refs=refs(model), **SCALING)
    E = float(r["energy"])
    assert abs(float(r["energies"].sum()) - E) <= 1e-10 * abs(E)
    W, Ws = r["virials"].sum(0), r["strain_virial"]
    assert float((W - Ws).abs().max()) <= 1e-10 * float(Ws.abs().max())
    # the oracle's geometry is that of potential_ref: same energy and stress
    if family == "chgnet":
        from oracle.chgnet_ref import potential_ref

        Eo, _F, So, _site = potential_ref(model_of(family), atoms, element_refs=refs(model), dtype=torch.float64,
                                          **SCALING)
    else:
        from oracle.tensornet_ref import potential_ref

        Eo, _F, So = potential_ref(model_of(family), atoms, element_refs=refs(model), dtype=torch.float64, **SCALING)
    assert abs(float(Eo) - E) <= 1e-10 * abs(E)
    assert float((So - r["stress"]).abs().max()) <= 1e-10 * float(So.abs().max())
    assert float((r["virials"].sum(0) / atoms.get_volume() * GPA_PER_EVA3 - So).abs().max()) <= 1e-9 * float(
        So.abs().max())


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("structure", list(STRUCTURES))
def test_translation_leaves_per_atom_values_unchanged(family, structure):
    atoms = STRUCTURES[structure]()
    model = model_of(family)
    r0 = atomic_ref(model, atoms, **SCALING)
    shifted = SimpleAtoms(atoms.get_chemical_symbols(), atoms.get_positions() + np.array([0.37, -1.21, 2.45]),
                          atoms.get_cell())
    r1 = atomic_ref(model, shifted, **SCALING)
    assert float((r0["energies"] - r1["energies"]).abs().max()) < 1e-9 * max(1.0, float(r0["energies"].abs().max()))
    assert float((r0["virials"] - r1["virials"]).abs().max()) < 1e-9 * max(1.0, float(r0["virials"].abs().max()))


# ---------------------------------------------------------------------------------------------- ASE calculator
try:
    import ase  # noqa: F401
except ImportError:
    sys.path.insert(0, os.path.join(HERE, "stubs"))

import distmlip_b200.implementations.matgl.ase as mase  # noqa: E402
from distmlip_b200.implementations.matgl.pes import Potential_Dist  # noqa: E402


class AtomicDouble(Potential_Dist):
    """Potential_Dist double with the per-atom outputs of calc_atomic: random per-atom energies and (non-symmetric)
    per-atom stresses whose sums are the returned energy and stress"""

    def __init__(self, n, calc_atomic, seed=0):
        rng = np.random.default_rng(seed)
        self.calc_forces = self.calc_stresses = True
        self.calc_hessian = self.calc_site_wise = False
        self.calc_atomic = calc_atomic
        self._e = rng.normal(-4.0, 0.3, n)
        self._s = rng.normal(0.0, 2.0, (n, 3, 3)).astype(np.float32)
        self.atomic_energies = self.atomic_stresses = None

    def forward(self, atoms, state_attr=None, tol=1e-8):
        if self.calc_atomic:
            self.atomic_energies = torch.from_numpy(self._e.copy())
            self.atomic_stresses = torch.from_numpy(self._s.copy())
        n = len(self._e)
        return (torch.tensor([self._e.sum()], dtype=torch.float64), torch.zeros(n, 3, dtype=torch.float32),
                torch.from_numpy(self._s.astype(np.float64).sum(0).astype(np.float32)), None)


def test_calculator_energies_and_stresses():
    atoms = si_diamond(1)
    n = len(atoms)
    cls_props = mase.PESCalculator_Dist.implemented_properties
    off = mase.PESCalculator_Dist(potential=AtomicDouble(n, calc_atomic=False))
    off.calculate(atoms, ["energy", "forces", "stress"])
    assert "energies" not in off.results and "stresses" not in off.results
    assert tuple(off.implemented_properties) == cls_props
    with pytest.raises(NotImplementedError):
        off.calculate(atoms, ["energies"])
    for use_voigt in (False, True):
        calc = mase.PESCalculator_Dist(potential=AtomicDouble(n, calc_atomic=True), use_voigt=use_voigt,
                                       stress_unit="eV/A3", stress_weight=2.0)
        assert "energies" in calc.implemented_properties and "stresses" in calc.implemented_properties
        calc.calculate(atoms, ["energy", "energies", "stresses"])
        r = calc.results
        assert r["energies"].shape == (n,) and abs(r["energies"].sum() - r["energy"]) <= 1e-12 * abs(r["energy"])
        assert r["stresses"].shape == ((n, 6) if use_voigt else (n, 3, 3))
        assert r["stress"].shape == ((6,) if use_voigt else (3, 3))
        tot = r["stresses"].astype(np.float64).sum(0)
        assert np.abs(tot - r["stress"]).max() <= 1e-5 * np.abs(r["stress"]).max()
    # the class attribute stays the reference's tuple
    assert mase.PESCalculator_Dist.implemented_properties == cls_props
    assert cls_props == ("energy", "free_energy", "forces", "stress", "hessian", "magmoms")


# ------------------------------------------------------------------ the GPU tolerances against routing bugs
# A kernel that adds an edge's half (or an atom's energy) to the wrong atom keeps both sum rules; only the per-atom
# comparison of tests/test_gpu_atomic.py sees it.  Its tolerances must stay far below what such bugs do.  The bugs are
# built from the oracle's per-edge halves in destination-sorted order (oracle.atomic_ref.routing_mutants); the
# 4000-atom GPU test repeats this in the engine's own edge order.
def gpu_structures():
    from tests.test_gpu_atomic import STRUCTURES, calculator_cell, irregular, slab

    return dict(STRUCTURES, slab=slab, calculator=calculator_cell, irregular=irregular)


@pytest.mark.parametrize("family", ["chgnet", "tensornet"])
@pytest.mark.parametrize("structure", ["diamond64", "diamond512", "rough", "slab", "calculator", "irregular"])
def test_gpu_tolerances_are_far_below_routing_bugs(family, structure):
    from oracle.atomic_ref import routing_mutants
    from tests.test_gpu_atomic import TOL_EPS, TOL_W

    # fp32 round-off, not accuracy targets: no looser than 1e-3 of max |w| and 2e-6 eV, whatever the margins below allow
    assert TOL_W[family] <= 1e-3 and TOL_EPS <= 2e-6
    atoms = gpu_structures()[structure]()
    model = model_of(family)
    r = atomic_ref(model, atoms, element_refs=refs(model), edges=True, **SCALING)
    w, src, dst, half = r["virials"], r["edge_src"], r["edge_dst"], r["edge_half"]
    bound = TOL_W[family] * float(w.abs().max())  # eV: the largest per-atom virial error the GPU tests accept
    errs = {name: float((wm - w).abs().max()) for name, wm in routing_mutants(src, dst, half, len(atoms)).items()}
    if family == "chgnet":
        # CHGNet's per-atom virials are symmetric to 1e-4 of max |w|: only TensorNet can show a transposition
        assert errs.pop("src_transposed") < 1e-3 * float(w.abs().max())
    for name, err in errs.items():
        assert err >= 10 * bound, (name, err, bound)
    # a single misrouted edge of median size is 10x above the tolerance
    edge = half.abs().amax((1, 2))
    assert bound <= 0.1 * float(edge.median()), (bound, float(edge.median()))
    # an atom's energy on one of its neighbours: 10x above the tolerance for 90 % of the edges
    eps = r["energies"]
    assert TOL_EPS <= 0.1 * float((eps[src] - eps[dst]).abs().quantile(0.1))
