"""GPU: TensorNet at a size where the persistent wgmma row GEMM (k_gemm_wg, csrc/kernels_wg.cu) loops.

k_gemm_wg launches at most two CTAs per SM and each CTA walks the 128-row tiles with a stride of the grid, prefetching
its next tile.  In the smaller TensorNet tests every CTA of the edge MLP gets at most one tile, so the loop and the
prefetch never run; this holds in particular for the SiLU / SiLU' epilogues (EPI = 1, 2) that only TensorNet uses.  The
4000-atom cell here has about 100 k edges, ~780 edge tiles, more than the resident CTAs of any k_gemm_wg shape."""
import os

import numpy as np
import pytest
import torch

from distmlip_b200.structures import rough_cell
from tests.test_gpu_tensornet import check_efs, mixed, oracle_efs, set_structure, tn_engine
from tests.test_oracle_tensornet import make_tn

pytestmark = pytest.mark.gpu
SCALING = dict(data_mean=0.7, data_std=1.3)
TILE_ROWS = 128   # rows per k_gemm_wg tile
CTAS_PER_SM = 2   # the most k_gemm_wg CTAs per SM: `per_sm` of launch_gemm_wg_t (csrc/kernels_wg.cu)


@pytest.fixture(scope="module")
def atoms():
    return mixed(rough_cell(4000, seed=11), other="Ge", every=2)


@pytest.fixture(scope="module")
def model():
    return make_tn(seed=3, scale=1.5)


def refs(model):
    return np.linspace(-0.5, 0.5, len(model.element_types))


def engine(model, ffma=False):
    """B2M_TN_FFMA=1 at construction selects the FP32-FFMA tile kernels (a plain grid over tiles) for this handle"""
    old = os.environ.get("B2M_TN_FFMA")
    try:
        os.environ["B2M_TN_FFMA"] = "1" if ffma else "0"
        return tn_engine(model, element_refs=refs(model), **SCALING)
    finally:
        if old is None:
            os.environ.pop("B2M_TN_FFMA", None)
        else:
            os.environ["B2M_TN_FFMA"] = old


def test_edge_tiles_outnumber_the_resident_ctas_and_match_the_oracle(atoms, model):
    eng = engine(model)
    set_structure(eng, model, atoms)
    tiles = eng.counts()["n_edges"] / TILE_ROWS
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"{eng.counts()['n_edges']} edges = {tiles:.0f} tiles, {CTAS_PER_SM * sms} resident CTAs at most")
    assert tiles > 2 * CTAS_PER_SM * sms  # every CTA of the largest grid walks at least two tiles
    ref = oracle_efs(model, atoms, element_refs=refs(model), **SCALING)
    e, f, s = check_efs(eng, model, atoms, ref)
    (E, F, S), _og = ref
    print(f"vs float64 oracle: |dE|/N {abs(e - float(E)) / len(atoms):.2e} eV, max|dF| {np.abs(f - F.numpy()).max():.2e} "
          f"eV/A, max|dS| {np.abs(s - S.numpy()).max():.2e} GPa")
    eng.close()


def test_wgmma_and_ffma_paths_agree(atoms, model):
    """the persistent wgmma path against the FFMA tiles at fp32 level: energy, forces, stress and per-atom values"""
    out = []
    for ffma in (False, True):
        eng = engine(model, ffma=ffma)
        set_structure(eng, model, atoms)
        eng.set_atomic(True)
        out.append(eng.compute(forces=True, stress=True) + eng.atomic())
        eng.close()
    (e1, f1, s1, eps1, w1), (e2, f2, s2, eps2, w2) = out
    n = len(atoms)
    de, df, ds = abs(e1 - e2) / n, np.abs(f1 - f2).max(), np.abs(s1 - s2).max()
    deps, dw = np.abs(eps1 - eps2).max(), np.abs(w1 - w2).max() / np.abs(w2).max()
    print(f"wgmma vs ffma: |dE|/N {de:.2e} eV, max|dF| {df:.2e} eV/A, max|dS| {ds:.2e} GPa, max|d eps| {deps:.2e} eV, "
          f"max|dw| / max|w| {dw:.2e}")
    # observed on an H100, largest of three runs: 6.9e-10 eV, 1.2e-7 eV/A, 1.5e-8 GPa, 9.7e-8 eV and 1.6e-6
    assert de < 5e-9 and df < 1e-6 and ds < 1.5e-7
    assert deps < 8e-7 and dw < 1e-5
