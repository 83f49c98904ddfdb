"""Scatter phase of the atom-conv and line-graph kernels (kernels.cu: scatter_rows): segmented sums over runs of equal
destination / out-bond / centre indices, reduced per thread over a few consecutive rows of a 128-row tile.

A run that straddles a thread's row boundary or a tile boundary is reduced in parts, and a partial last tile has rows
with no index at all; every row must still land exactly once.  Checked through energies, forces and stress against the
oracle at sizes where the persistent kernels loop (more tiles than SMs), on the degree-imbalanced rough cell (runs of
every length from 0 upwards) and on cells whose edge and angle counts are not multiples of the tile height, and across
partitionings of one cell (different row orders and run cuts, halo bonds, layers without an atom gradient).
"""
import pytest
import torch

from distmlip_b200.structures import rough_cell, si_diamond
from oracle.chgnet_ref import potential_ref
from tests._util import make_model

pytestmark = pytest.mark.gpu
TOL_E, TOL_F, TOL_S = 2e-7, 3e-6, 3e-6  # as tests/test_gpu_group.py
TILE = 128


def potential(devices):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    dm = CHGNet_Dist.from_existing(make_model())
    dm.enable_distributed_mode(devices)
    return dm, Potential_Dist(model=dm)


def assert_kernels_loop_with_partial_tile(counts):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for what in ("n_edges", "n_angles"):
        n = counts[what]
        assert n % TILE != 0, (what, n)
        assert (n + TILE - 1) // TILE > sms, (what, n, sms)


@pytest.mark.parametrize("atoms", [
    pytest.param(lambda: rough_cell(2400, seed=11), id="rough"),
    pytest.param(lambda: si_diamond(5, nz=11, seed=3), id="diamond"),
])
def test_one_partition_matches_oracle(atoms):
    atoms = atoms()
    dm, pot = potential([0])
    E, F, S, _ = pot(atoms)
    assert_kernels_loop_with_partial_tile(dm._engine.counts())
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S
    dm._engine.close()


def test_one_and_three_partitions_agree():
    atoms = rough_cell(3600, seed=4, aspect=(1, 1, 6))
    dm1, pot1 = potential([0])
    dm3, pot3 = potential([0, 0, 0])
    E1, F1, S1, _ = pot1(atoms)
    E3, F3, S3, _ = pot3(atoms)
    assert_kernels_loop_with_partial_tile(dm1._engine.counts())
    assert dm3._engine.counts()["n_bond_halo"] > 0
    assert abs(E1.item() - E3.item()) / len(atoms) < 1e-7
    assert (F1 - F3).abs().max().item() < 2e-6 and (S1 - S3).abs().max().item() < 2e-6
    dm1._engine.close(), dm3._engine.close()
