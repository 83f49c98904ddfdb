"""Rank-9 radial products of the atom-conv kernels on the tensor cores (kernels.cu: radial_mma): be.M^T in the first
layer of both kernels, w_ab = be.W_ab^T in the forward gates and the backward's elementwise reverse, and dE/dd as one
scalar per row from dbe.W_ab^T and dbe.M^T.

Checked through energies, forces and stress against the oracle where the radial terms dominate: cells compressed and
stretched by about 10 % put many edges in the envelope region near the cutoff, and move bonds across the bond cutoff,
where rows switch between Q[bond] and M.be; mixed species; edge counts that are not multiples of the 128-row tile; one
and three partitions of one cell.
"""
import numpy as np
import pytest

from distmlip_b200.structures import SimpleAtoms, si_diamond
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


def strained(cells, scale, seed, mixed, nz=None):
    atoms = si_diamond(cells, seed=seed, nz=nz)
    sym = atoms.get_chemical_symbols()
    if mixed:
        sym = ["Ge" if x < 0.3 else "Si" for x in np.random.default_rng(seed).random(len(atoms))]
    return SimpleAtoms(sym, atoms.get_positions() * scale, atoms.get_cell() * scale)


@pytest.mark.parametrize("scale", [0.9, 1.1], ids=["compressed", "stretched"])
@pytest.mark.parametrize("mixed", [False, True], ids=["si", "si_ge"])
def test_strained_cell_matches_oracle(scale, mixed):
    atoms = strained(4, scale, seed=7, mixed=mixed)
    dm, pot = potential([0])
    E, F, S, _ = pot(atoms)
    assert dm._engine.counts()["n_edges"] % TILE != 0
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S
    dm._engine.close()


def test_one_and_three_partitions_agree_strained():
    atoms = strained(3, 1.08, seed=5, mixed=True, nz=10)  # 19 A slabs
    dm1, pot1 = potential([0])
    dm3, pot3 = potential([0, 0, 0])
    E1, F1, S1, _ = pot1(atoms)
    E3, F3, S3, _ = pot3(atoms)
    assert dm1._engine.counts()["n_edges"] % TILE != 0
    assert abs(E1.item() - E3.item()) / len(atoms) < 1e-7
    assert (F1 - F3).abs().max().item() < 2e-6 and (S1 - S3).abs().max().item() < 2e-6
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E3.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F3 - Fo).abs().max().item() < TOL_F and (S3 - So).abs().max().item() < TOL_S
    dm1._engine.close(), dm3._engine.close()
