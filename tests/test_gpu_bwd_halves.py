"""Backward tile kernels one 64-row half at a time (kernels.cu: k_atomconv_bwd, k_line_bwd): the recompute parks the
second layer's outputs in the exchange tile, and the reverse reads them back and runs its elementwise step, g.W2 and
the radial terms half by half, with all of a half's upstream loads issued together.

The wgmma products are warpgroup-collective, so they must be issued for both halves even where a partial last tile
leaves half 1 empty (1-63 valid rows) or only partly filled (65-127).  Checked through energies, forces and stress
against the oracle at edge and angle counts with each kind of last tile, at sizes where the persistent kernels loop
(more tiles than SMs), on the rough cell (bond rows fed by Q next to radial rows, runs of every length), and on a
strained mixed Si/Ge cell on one and three partitions.
"""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.chgnet_ref import potential_ref
from tests._util import make_model

pytestmark = pytest.mark.gpu
TOL_E, TOL_F, TOL_S = 2e-7, 3e-6, 3e-6  # as tests/test_gpu_scatter_runs.py
TILE = 128


def potential(devices):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    dm = CHGNet_Dist.from_existing(make_model())
    dm.enable_distributed_mode(devices)
    return dm, Potential_Dist(model=dm)


def assert_kernels_loop(counts, last_rows=None):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for what in ("n_edges", "n_angles"):
        n = counts[what]
        assert (n + TILE - 1) // TILE > sms, (what, n, sms)
        if last_rows is not None:
            assert n % TILE in last_rows, (what, n)


def check_against_oracle(atoms, last_rows=None):
    dm, pot = potential([0])
    E, F, S, _ = pot(atoms)
    assert_kernels_loop(dm._engine.counts(), last_rows)
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S
    dm._engine.close()


# 5 x 5 x 11 cells, seed 0: 61 572 edges (last tile 4 rows), 26 392 angles (24 rows)
def test_last_tile_half_one_empty():
    check_against_oracle(si_diamond(5, nz=11, seed=0), last_rows=range(1, 64))


# 5 x 5 x 9 cells, seed 0: 50 380 edges (last tile 76 rows), 21 600 angles (96 rows)
def test_last_tile_half_one_partial():
    check_against_oracle(si_diamond(5, nz=9, seed=0), last_rows=range(65, 128))


def test_rough_cell():
    check_against_oracle(rough_cell(2400, seed=21))


def test_strained_si_ge_one_and_three_partitions():
    base = si_diamond(5, nz=10, seed=9)
    sym = ["Ge" if x < 0.4 else "Si" for x in np.random.default_rng(9).random(len(base))]
    atoms = SimpleAtoms(sym, base.get_positions() * 0.95, base.get_cell() * 0.95)
    dm1, pot1 = potential([0])
    dm3, pot3 = potential([0, 0, 0])
    E1, F1, S1, _ = pot1(atoms)
    E3, F3, S3, _ = pot3(atoms)
    assert_kernels_loop(dm1._engine.counts())
    assert dm3._engine.counts()["n_bond_halo"] > 0
    assert abs(E1.item() - E3.item()) / len(atoms) < 1e-7
    assert (F1 - F3).abs().max().item() < 2e-6 and (S1 - S3).abs().max().item() < 2e-6
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E1.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F1 - Fo).abs().max().item() < TOL_F and (S1 - So).abs().max().item() < TOL_S
    dm1._engine.close(), dm3._engine.close()
