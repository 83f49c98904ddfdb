"""GPU: TensorNet at a size where the persistent wgmma row GEMM (k_gemm_wg, csrc/kernels_wg.cu) loops.

k_gemm_wg launches at most two CTAs per SM and each CTA walks the 128-row tiles with a stride of the grid, prefetching
its next tile.  In the smaller TensorNet tests every CTA of the edge MLP gets at most one tile, so the loop and the
prefetch never run; this holds in particular for the SiLU / SiLU' epilogues (EPI = 1, 2) that only TensorNet uses.  The
4000-atom cell here has about 100 k edges, ~780 edge tiles, more than the resident CTAs of any k_gemm_wg shape."""
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


def test_edge_tiles_outnumber_the_resident_ctas_and_match_the_oracle(atoms, model):
    eng = tn_engine(model, element_refs=refs(model), **SCALING)
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
