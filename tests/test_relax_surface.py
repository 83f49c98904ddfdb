"""Batched relaxation, Python surface (CPU): Relaxer.relax_batch and ScaleShiftMACE_Dist.relax_batch hand the
concatenated batch to one b2m_relax_batch, split its results per structure in order, leave the inputs untouched, and
refuse what the device loop cannot do before the engine is touched.  A stand-in engine replaces the GPU one here; the
real engine runs in tests/test_gpu_relax.py."""
import numpy as np
import pytest

from tests.test_batch_surface import BatchEngine, batch, stand_in  # noqa: F401  (puts the ASE stand-in on the path)

from distmlip_b200 import _lib  # noqa: E402
from distmlip_b200.implementations.mace.models import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.implementations.matgl.ase import Relaxer  # noqa: E402
from distmlip_b200.implementations.matgl.models.chgnet import CHGNet_Dist  # noqa: E402
from distmlip_b200.implementations.matgl.pes import Potential_Dist  # noqa: E402
from distmlip_b200.structures import SimpleAtoms  # noqa: E402

GPA_PER_EVA3 = 160.21766208


class RelaxEngine(BatchEngine):
    """relax_batch moves every atom by +1 A along x and scales every cell by 2; structure s takes s + 1 steps, converges
    when s is even, and has energies s + 0.5 - 0.1 t per evaluation t"""

    def relax_batch(self, natoms, cart, lattices, species, pbc, **kw):
        self.calls.append("relax_batch")
        self.kw = kw
        self.n, self.species, self.pbc = np.asarray(natoms), species, pbc
        S = len(natoms)
        steps = np.arange(S) + 1
        tr = np.full((S, kw["steps"] + 1), np.nan)
        for s in range(S):
            tr[s, :steps[s] + 1] = s + 0.5 - 0.1 * np.arange(steps[s] + 1)
        return dict(cart=cart + [1.0, 0.0, 0.0], lattices=lattices * 2, energies=np.arange(S) + 0.5,
                    forces=(-cart).astype(np.float32), stress=np.repeat(np.eye(3)[None], S, 0).astype(np.float32) * 3,
                    steps=steps.astype(np.int32), converged=steps % 2 == 1, trace=tr if kw["trace"] else None)


def check(atoms, before, out):
    assert len(out) == len(atoms)
    for k, (a, (x, c), o) in enumerate(zip(atoms, before, out)):
        np.testing.assert_array_equal(a.get_positions(), x)  # inputs untouched
        np.testing.assert_array_equal(a.get_cell(), c)
        fs = o["final_structure"]
        assert fs is not a
        np.testing.assert_array_equal(fs.get_positions(), x + [1.0, 0.0, 0.0])
        np.testing.assert_array_equal(fs.get_cell(), 2 * c)
        assert o["energy"] == k + 0.5 and o["steps"] == k + 1 and o["converged"] == (k % 2 == 0)
        np.testing.assert_array_equal(o["forces"], -x.astype(np.float32))
        np.testing.assert_allclose(o["stress"], 3 * np.eye(3) / GPA_PER_EVA3)
        np.testing.assert_allclose(o["energies"], k + 0.5 - 0.1 * np.arange(k + 2))


def test_relaxer_splits_per_structure():
    eng = RelaxEngine()
    r = Relaxer(potential=Potential_Dist(model=stand_in(CHGNet_Dist, eng)), relax_cell=True)
    atoms = [a for a in batch((7, 2, 13)) if a.get_pbc().all()] + [batch((5,), seed=3)[0]]
    before = [(a.get_positions().copy(), a.get_cell().copy()) for a in atoms]
    out = r.relax_batch(atoms, fmax=0.05, steps=9, params_asecellfilter={"scalar_pressure": 0.01}, dt=0.05, Nmin=3)
    check(atoms, before, out)
    assert eng.calls.index("finalize") < eng.calls.index("relax_batch")
    kw = eng.kw
    assert kw["fmax"] == 0.05 and kw["steps"] == 9 and kw["relax_cell"] and kw["scalar_pressure"] == 0.01
    assert kw["stress_weight"] == 1 / 160.21766208 and kw["dt"] == 0.05 and kw["Nmin"] == 3
    assert list(eng.n) == [len(a) for a in atoms]


def test_mace_relax_batch_positions_only_keeps_slabs():
    eng = RelaxEngine()
    model = stand_in(ScaleShiftMACE_Dist, eng)
    atoms = batch((5, 1, 9))  # the second is a slab
    before = [(a.get_positions().copy(), a.get_cell().copy()) for a in atoms]
    out = model.relax_batch(atoms, fmax=0.2, steps=4, relax_cell=False, maxstep=0.1)
    check(atoms, before, out)
    assert not eng.kw["relax_cell"] and eng.kw["maxstep"] == 0.1 and eng.kw["scalar_pressure"] == 0.0
    assert eng.pbc.tolist() == [[1, 1, 1], [1, 1, 0], [1, 1, 1]]


def test_without_the_energy_trace():
    eng = RelaxEngine()
    out = stand_in(ScaleShiftMACE_Dist, eng).relax_batch(batch((5, 3)), steps=4, relax_cell=False, trace=False)
    assert eng.kw["trace"] is False and [o["energies"] for o in out] == [None, None]


def test_refusals_before_the_engine_is_touched():
    eng = RelaxEngine()
    pot = Potential_Dist(model=stand_in(CHGNet_Dist, eng))
    periodic = [batch((4,))[0]]
    with pytest.raises(NotImplementedError, match="FIRE only"):
        Relaxer(potential=pot, optimizer="BFGS").relax_batch(periodic)
    r = Relaxer(potential=pot)
    with pytest.raises(NotImplementedError, match="Frechet cell filter only"):
        r.relax_batch(periodic, ase_cellfilter="Exp")
    with pytest.raises(NotImplementedError, match="scalar_pressure"):
        r.relax_batch(periodic, params_asecellfilter={"hydrostatic_strain": True})
    with pytest.raises(TypeError, match="downhill_check"):
        r.relax_batch(periodic, downhill_check=True)
    with pytest.raises(ValueError, match="empty batch"):
        r.relax_batch([])
    with pytest.raises(ValueError, match="structure 1: relax_cell needs a cell periodic"):
        r.relax_batch(batch((4, 5)))
    for group, world in ((True, 2), (False, 2)):
        with pytest.raises(NotImplementedError, match="one GPU and one partition"):
            Relaxer(potential=Potential_Dist(model=stand_in(CHGNet_Dist, BatchEngine(group, world)))).relax_batch(
                periodic)
    with pytest.raises(NotImplementedError, match="heat flux"):
        Relaxer(potential=Potential_Dist(model=stand_in(CHGNet_Dist, eng), calc_heat_flux=True)).relax_batch(periodic)
    mace = stand_in(ScaleShiftMACE_Dist, eng)
    with pytest.raises(TypeError, match="downhill_check"):
        mace.relax_batch(periodic, downhill_check=True)
    with pytest.raises(ValueError, match="empty batch"):
        mace.relax_batch([])
    alien = [SimpleAtoms(["Si", "Ge"], np.eye(2, 3), np.eye(3) * 5)]
    with pytest.raises(KeyError, match="not in model.element_types"):
        mace.relax_batch(alien)
    assert eng.calls == []


def test_engine_refuses_unknown_fire_constants():
    with pytest.raises(TypeError, match="unknown FIRE parameters"):
        _lib.Engine.relax_batch(None, [1], np.zeros((1, 3)), np.eye(3)[None], [0], [[1, 1, 1]], downhill_check=True)
