"""Batched evaluation, Python surface (CPU): Potential_Dist.forward_batch and ScaleShiftMACE_Dist.evaluate_batch split the
concatenated results of one b2m_compute_batch per structure, in order, with the shapes and types of forward / evaluate,
and refuse what a batch cannot do before the engine is touched.  A stand-in engine replaces the GPU one here; the real
engine runs in tests/test_gpu_batch.py.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
try:
    import ase  # noqa: F401
except ImportError:
    sys.path.insert(0, os.path.join(HERE, "stubs"))
    import ase  # noqa: F401

from distmlip_b200.implementations.mace.models import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.implementations.matgl.models.chgnet import CHGNet_Dist  # noqa: E402
from distmlip_b200.implementations.matgl.models.tensornet import TensorNet_Dist  # noqa: E402
from distmlip_b200.implementations.matgl.pes import Potential_Dist  # noqa: E402
from distmlip_b200.structures import SimpleAtoms  # noqa: E402

GPA_PER_EVA3 = 160.21766208


class BatchEngine:
    """Stand-in for _lib.Engine: every result is a function of the concatenated inputs that names its atom or
    structure (forces = -positions, energy of structure s = s + 0.5, per-atom energy = species + 0.25, ...), so a
    split in the wrong place or order shows."""

    def __init__(self, group=False, world=1):
        self.group, self.world = group, world
        self.calls = []

    def __getattr__(self, name):  # set_scaling, set_element_refs, finalize, set_heat_flux: recorded, no effect
        if name.startswith("__"):
            raise AttributeError(name)
        return lambda *a, **k: self.calls.append(name)

    def set_structures(self, natoms, cart, cells, species, pbc, tol=1e-8):
        self.calls.append("set_structures")
        self.n, self.cart, self.cells, self.species, self.pbc = np.asarray(natoms), cart, cells, species, pbc
        assert cart.shape == (self.n.sum(), 3) and species.shape == (self.n.sum(),) and cells.shape == (len(natoms), 3, 3)

    def compute_batch(self, forces=True, stress=True):
        self.calls.append("compute_batch")
        S = len(self.n)
        e = np.arange(S) + 0.5
        f = (-self.cart).astype(np.float32) if forces else None
        s = (self.cells * 2).astype(np.float32) if stress else None
        return e, f, s

    def atomic(self, virials=True):
        w = np.repeat(self.cart[:, :, None], 3, axis=2).astype(np.float32) if virials else None
        return self.species + 0.25, w

    def sitewise(self):
        return self.cart[:, 0].astype(np.float32)


def stand_in(cls, eng, elements=("Si", "O")):
    m = cls.__new__(cls)
    m.__dict__.update(dist_enabled=True, _engine=eng, gpus=["cuda:0"], element_to_index={s: i for i, s in enumerate(elements)},
                      element_types=tuple(elements), _engine_finalized=False, cutoff=5.0, three_body_cutoff=3.0,
                      _rank=0, _world=1)
    return m


def batch(sizes=(7, 2, 13), seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k, n in enumerate(sizes):
        cell = np.eye(3) * (4.0 + k)
        sym = ["O" if (i + k) % 3 == 0 else "Si" for i in range(n)]
        out.append(SimpleAtoms(sym, rng.random((n, 3)) * 4.0, cell, pbc=(True, True, k % 2 == 0)))
    return out


def test_forward_batch_splits_per_structure_in_order():
    eng = BatchEngine()
    model = stand_in(CHGNet_Dist, eng)
    pot = Potential_Dist(model=model, calc_site_wise=True, calc_atomic=True)
    atoms = batch()
    out = pot.forward_batch(atoms)
    assert eng.calls.index("finalize") < eng.calls.index("set_structures") < eng.calls.index("compute_batch")
    assert list(eng.n) == [len(a) for a in atoms]
    assert eng.pbc.tolist() == [[1, 1, 1], [1, 1, 0], [1, 1, 1]]
    assert len(out) == len(atoms)
    for k, (a, o) in enumerate(zip(atoms, out)):
        assert len(o) == 5
        E, F, S, H, site = o
        assert E.dtype == torch.float64 and E.shape == (1,) and float(E) == k + 0.5
        assert F.dtype == torch.float32 and F.shape == (len(a), 3)
        np.testing.assert_array_equal(F.numpy(), -a.get_positions().astype(np.float32))
        assert S.shape == (3, 3) and np.array_equal(S.numpy(), 2 * np.array(a.get_cell(), dtype=np.float32))
        assert H is None
        assert site.shape == (len(a), 1) and np.array_equal(site.numpy()[:, 0], a.get_positions()[:, 0].astype(np.float32))
        sp = np.array([0 if s == "Si" else 1 for s in a.get_chemical_symbols()])
        assert pot.atomic_energies[k].dtype == torch.float64
        np.testing.assert_array_equal(pot.atomic_energies[k].numpy(), sp + 0.25)
        assert pot.atomic_stresses[k].dtype == torch.float32 and pot.atomic_stresses[k].shape == (len(a), 3, 3)
        want = np.repeat(a.get_positions()[:, :, None], 3, axis=2) * GPA_PER_EVA3 / a.get_volume()
        np.testing.assert_allclose(pot.atomic_stresses[k].numpy(), want, rtol=1e-6)


def test_forward_batch_without_site_wise_or_backward():
    eng = BatchEngine()
    pot = Potential_Dist(model=stand_in(TensorNet_Dist, eng), calc_forces=False, calc_stresses=False, calc_atomic=True)
    out = pot.forward_batch(batch((3, 4)))
    assert [len(o) for o in out] == [4, 4]
    assert all(o[1] is None and o[2] is None for o in out)
    assert pot.atomic_stresses == [None, None] and [len(x) for x in pot.atomic_energies] == [3, 4]


def test_evaluate_batch_returns_evaluate_tuples():
    eng = BatchEngine()
    model = stand_in(ScaleShiftMACE_Dist, eng)
    atoms = batch((5, 1, 9))
    out = model.evaluate_batch(atoms, atomic=True)
    for k, (a, (e, f, s, ae, av)) in enumerate(zip(atoms, out)):
        assert isinstance(e, float) and e == k + 0.5
        assert f.shape == (len(a), 3) and s.shape == (3, 3) and ae.shape == (len(a),) and av.shape == (len(a), 3, 3)
        np.testing.assert_array_equal(f, -a.get_positions().astype(np.float32))
    e, f, s, ae, av = model.evaluate_batch(atoms, forces=False, stress=False)[2]
    assert f is None and s is None and ae is None and av is None


@pytest.mark.parametrize("call", ["forward_batch", "evaluate_batch"])
def test_refusals_before_the_engine_is_touched(call):
    def run(eng, atoms_list, **kw):
        if call == "forward_batch":
            return Potential_Dist(model=stand_in(CHGNet_Dist, eng), **kw).forward_batch(atoms_list)
        return stand_in(ScaleShiftMACE_Dist, eng).evaluate_batch(atoms_list)

    eng = BatchEngine()
    with pytest.raises(ValueError, match="empty batch"):
        run(eng, [])
    for group, world in ((True, 2), (False, 2)):
        with pytest.raises(NotImplementedError, match="one GPU and one partition"):
            run(BatchEngine(group, world), batch())
    alien = batch((4, 3))
    alien[1] = SimpleAtoms(["Si", "Ge", "Si"], alien[1].get_positions(), alien[1].get_cell())
    with pytest.raises(KeyError, match="not in model.element_types"):
        run(eng, alien)
    if call == "forward_batch":
        with pytest.raises(NotImplementedError, match="heat flux"):
            run(eng, batch(), calc_heat_flux=True)
    assert eng.calls == []
