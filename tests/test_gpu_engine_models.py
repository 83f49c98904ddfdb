"""GPU: what the engine's shared frame does the same way for every model.  b2m_release_workspace frees each model's
workspace and the frame's per-structure buffers, and the handle evaluates again after the next set_structure, for
TensorNet and MACE (0e and 0e+1o hidden features) on one partition and on a two-partition group (CHGNet:
tests/test_gpu_parity.py).  The capability guards keep refusing what a model does not have."""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import si_diamond
from tests._util import engine_from_model, make_model
from tests.test_gpu_parity import run_engine
from tests.test_gpu_tensornet import mixed as tn_mixed, set_structure, tn_engine
from tests.test_oracle_tensornet import make_tn

pytestmark = pytest.mark.gpu

PARTS = [1, 2]


def devices(parts):
    return 0 if parts == 1 else [0] * parts


def mace_dist(max_L, parts):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist
    from tests.test_gpu_mace_equivariant import model

    d = ScaleShiftMACE_Dist.from_existing(model(seed=11, max_L=max_L))
    d.enable_distributed_mode([0] * parts)
    return d


def release_then_reuse(eng, evaluate, natoms):
    """evaluate, release, check that memory came back and that compute refuses, evaluate again"""
    from distmlip_b200._lib import B2MError

    e1, f1, s1 = evaluate()
    used = torch.cuda.mem_get_info()[0]
    eng.release_workspace()
    assert torch.cuda.mem_get_info()[0] > used
    with pytest.raises(B2MError):
        eng.compute(True, True)
    e2, f2, s2 = evaluate()
    assert abs(e1 - e2) / natoms < 2e-8 and np.abs(f1 - f2).max() < 1e-6
    assert np.abs(s1 - s2).max() < 1e-6


@pytest.mark.parametrize("parts", PARTS)
def test_tensornet_release_workspace_then_reuse(parts):
    model = make_tn(seed=4, scale=1.5)
    atoms = tn_mixed(si_diamond(4, sigma=0.15, seed=3, nz=8))
    eng = tn_engine(model, device=devices(parts))

    def evaluate():
        set_structure(eng, model, atoms)
        return eng.compute(forces=True, stress=True)

    release_then_reuse(eng, evaluate, len(atoms))
    eng.close()


@pytest.mark.parametrize("max_L", [0, 1], ids=["0e", "0e+1o"])
@pytest.mark.parametrize("parts", PARTS)
def test_mace_release_workspace_then_reuse(max_L, parts):
    from tests.test_gpu_mace_equivariant import mixed

    d = mace_dist(max_L, parts)
    atoms = mixed(si_diamond(4, nz=8, seed=6))

    def evaluate():
        return d.evaluate(atoms)[:3]

    release_then_reuse(d._engine, evaluate, len(atoms))


def test_capability_guards():
    from distmlip_b200._lib import B2MError

    chg_model = make_model()
    chg = engine_from_model(chg_model)
    atoms = si_diamond(2, seed=1)
    run_engine(chg, chg_model, atoms)

    tn_model = make_tn(seed=2, scale=1.5)
    tn = tn_engine(tn_model)
    tn_atoms = tn_mixed(si_diamond(2, sigma=0.15, seed=5))
    set_structure(tn, tn_model, tn_atoms)
    tn.compute(True, True)

    from tests.test_gpu_mace_equivariant import mixed

    d = mace_dist(1, 1)
    d.evaluate(mixed(si_diamond(2, seed=7)))
    mace = d._engine

    def refused(call, text):
        with pytest.raises(B2MError) as ei:
            call()
        assert text in str(ei.value), str(ei.value)

    refused(lambda: mace.set_scaling(0.0, 1.0), "a MACE model carries its own scale and shift (scale_shift)")
    refused(lambda: mace.set_element_refs(np.zeros(3)),
            "a MACE model carries its own atomic energies (atomic_energies_fn)")
    site = "the site-wise readout belongs to CHGNet (TensorNet and MACE have none)"
    refused(tn.sitewise, site)
    refused(mace.sitewise, site)
    assert chg.sitewise().shape == (len(atoms),)
    for eng in (chg, tn, mace):
        refused(lambda: eng.debug_tensor("no_such_tensor"), "unknown debug tensor: no_such_tensor")
    chg.close()
    tn.close()
