"""Single-process multi-partition groups (b2m_create with ndev > 1): the reference's own usage,
`enable_distributed_mode([0, 1, ...])` from one Python process (examples/chgnet_example.ipynb cell 1; chgnet.py:455-549).

Device ordinals may repeat, so the whole graph-parallel path -- slab partition, halo sections, forward halo pushes into the
neighbour's rows, backward adjoint pushes + accumulate-into-owner, per-partition host threads and the event ordering --
runs on a ONE-GPU box ([0, 0], [0, 0, 0]) and is compared with the single-partition oracle (the arithmetic of the
distributed path is partition independent).  With >= 2 GPUs the same tests also run on distinct devices (peer access).
"""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from oracle.chgnet_ref import potential_ref
from tests._util import make_model

pytestmark = pytest.mark.gpu
TOL_E, TOL_F, TOL_S = 2e-7, 3e-6, 3e-6


def group_potential(devices, **kw):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    dm = CHGNet_Dist.from_existing(make_model())
    dm.enable_distributed_mode(devices)  # one process, several partitions
    return dm, Potential_Dist(model=dm, **kw)


def device_lists(n):
    out = [[0] * n]
    if torch.cuda.device_count() >= n:
        out.append(list(range(n)))
    return out


@pytest.mark.parametrize("nparts", [2, 3])
def test_group_matches_oracle(nparts):
    atoms = si_diamond(4, nz=4 * nparts, seed=3)  # 21.7 A slabs > 2 (r_cut + r_bond)
    Eo, Fo, So, siteo = potential_ref(make_model(), atoms, data_mean=0.5, data_std=1.5)
    for devs in device_lists(nparts):
        dm, pot = group_potential(devs, data_mean=0.5, data_std=1.5, calc_site_wise=True)
        E, F, S, _, site = pot(atoms)
        n = len(atoms)
        assert abs(E.item() - Eo.item()) / n < TOL_E, devs
        assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S, devs
        assert (site - siteo).abs().max().item() < 5e-6
        c = dm._engine.counts()
        assert c["world"] == nparts and c["n_halo"] > 0 and c["n_bond_halo"] > 0
        # a second evaluation on the resident graph reuses events and receive buffers: same numbers
        E2, _ms = dm._engine.compute_resident(2)
        assert abs(E2 - E.item()) / n < 2e-8  # fp32 atomics: run-to-run differences at round-off level
        dm._engine.close()


def test_group_irregular_structure_and_moving_atoms():
    """rough cell (destination runs of every length, uneven halo sections) and an MD-like sequence of structures on
    one group: graph rebuilt per call on every partition, event / buffer reuse across calls"""
    base = rough_cell(2400, seed=5, aspect=(1, 1, 4))
    dm, pot = group_potential([0, 0])
    rng = np.random.default_rng(0)
    pos = base.get_positions()
    for step in range(3):
        atoms = SimpleAtoms(base.get_chemical_symbols(), pos, base.get_cell())
        E, F, S, _ = pot(atoms)
        Eo, Fo, So, _ = potential_ref(make_model(), atoms)
        assert abs(E.item() - Eo.item()) / len(atoms) < TOL_E, step
        assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S, step
        pos = pos + rng.normal(0.0, 0.03, size=pos.shape)
    dm._engine.close()


def test_group_equals_single_partition_engine():
    atoms = si_diamond(5, nz=10, seed=9)  # 2000 atoms
    dm1, pot1 = group_potential([0])
    dm2, pot2 = group_potential([0, 0])
    E1, F1, S1, _ = pot1(atoms)
    E2, F2, S2, _ = pot2(atoms)
    assert abs(E1.item() - E2.item()) / len(atoms) < 1e-7
    assert (F1 - F2).abs().max().item() < 2e-6 and (S1 - S2).abs().max().item() < 2e-6
    dm1._engine.close(), dm2._engine.close()


def test_group_errors_come_back_from_the_partition_threads():
    from distmlip_b200._lib import B2MError

    dm, pot = group_potential([0, 0])
    with pytest.raises(B2MError) as ei:
        pot(si_diamond(4))  # 10.9 A slabs <= 2 (r_cut + r_bond): subgraph_creation_utils.c:1512-1529
    assert ei.value.code == -4 and "too close" in str(ei.value)
    E, F, S, _ = pot(si_diamond(4, nz=8, seed=1))  # the group stays usable
    assert np.isfinite(F.numpy()).all()
    dm._engine.close()


def test_group_partition_views_agree():
    """the reference keeps every partition's arrays on the host and its counters take a `partition` argument
    (dist.py:39-99, 462-551); in a single-process group the same questions are answered per partition (b2m_set_view):
    owned atoms partition the structure, what partition q lists "to p" is exactly p's halo section from q, in order."""
    atoms = si_diamond(4, nz=12, seed=7)
    dm, pot = group_potential([0, 0, 0])
    pot(atoms)
    d = pot.last_dist_info
    P = 3
    own = [d.partition_content(p, 0) for p in range(P)]
    assert sorted(np.concatenate(own).tolist()) == list(range(len(atoms)))
    assert sum(d.num_atoms(p) - d.num_atom_border_nodes(p) for p in range(P)) == len(atoms)
    for p in range(P):
        halo, howner = d.partition_content(p, 1), d.partition_content(p, 2)
        assert d.num_atom_border_nodes(p) == len(halo) and d.num_bond_border_nodes(p) > 0
        for q in range(P):
            if q == p:
                continue
            tl = d.partition_content(q, 6)
            assert np.array_equal(tl[tl[:, 0] == p, 1], halo[howner == q])
    text = repr(d)
    assert text.count("Partition ") == 3 and "border nodes" in text
    with pytest.raises(ValueError):
        d.num_atoms(5)
    dm._engine.close()


def test_group_triclinic_cell():
    """sheared cell, two partitions: slab walls in wrapped fractional coordinate of a non-orthogonal lattice"""
    a = si_diamond(4, nz=9, seed=15)
    lat = a.get_cell()
    lat[2, 0], lat[1, 0] = 3.0, 1.5
    atoms = SimpleAtoms(a.get_chemical_symbols(), a.get_scaled_positions() @ lat, lat)
    dm, pot = group_potential([0, 0])
    E, F, S, _ = pot(atoms)
    Eo, Fo, So, _ = potential_ref(make_model(), atoms)
    assert abs(E.item() - Eo.item()) / len(atoms) < TOL_E
    assert (F - Fo).abs().max().item() < TOL_F and (S - So).abs().max().item() < TOL_S
    dm._engine.close()


def _tensornet_potential(devices):
    from distmlip_b200.implementations.matgl import Potential_Dist, TensorNet_Dist
    from tests.test_oracle_tensornet import make_tn

    dm = TensorNet_Dist.from_existing(make_tn(seed=6, scale=1.5))
    dm.enable_distributed_mode(devices)
    return dm, Potential_Dist(model=dm)


@pytest.mark.parametrize("model", ["chgnet", "tensornet"])
@pytest.mark.parametrize("devices", [[0], [0, 0]])
def test_launch_count_is_the_kernels_the_device_ran(model, devices, tmp_path):
    """counts()["launches"] of an evaluation is the number of kernels it ran; in a group every partition's host thread
    counts its own launches only, however the partitions' evaluations overlap"""
    import json

    from torch.profiler import ProfilerActivity, profile

    dm, pot = group_potential(devices) if model == "chgnet" else _tensornet_potential(devices)
    pot(si_diamond(4, nz=8, seed=2))
    eng = dm._engine
    eng.compute_resident(1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.compute_resident(1)
    prof.export_chrome_trace(str(tmp_path / "trace.json"))
    events = json.loads((tmp_path / "trace.json").read_text())["traceEvents"]
    kernels = sum(1 for ev in events if ev.get("cat") == "kernel")  # memcpy / memset records are other categories
    assert kernels > 0 and eng.counts()["launches"] == kernels
    eng.close()
