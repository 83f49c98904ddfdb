"""MACE with the ZBL pair repulsion and the Agnesi distance transform on the H100 engine against the f64 oracle
(tests/mace_zbl_ref.py), for both hidden shapes, with the thresholds of test_gpu_mace*.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from distmlip_b200.structures import Z_OF, SimpleAtoms, si_diamond
from tests.mace_zbl_ref import atomic_virials_ref, potential_ref
from tests.test_oracle_mace_zbl import OPTIONS, close_contact, cluster, diamond64, dimer, mixed, model

pytestmark = pytest.mark.gpu

SHAPES = {"0e": False, "0e+1o": True}


def run(m, atoms, gpus=(0,)):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode(list(gpus))
    return d, d.evaluate(atoms, atomic=True)


def check(m, atoms, gpus=(0,), rel=False, virials=False):
    """the thresholds of test_gpu_mace.py; rel: plus 1e-5 of max |F| and of |E_pair| (close contacts, where fp32 carries
    pair energies of hundreds of eV)"""
    taps = {}
    E, F, S, eps = potential_ref(m, atoms)
    potential_ref(m, atoms, calc_forces=False, taps=taps)
    _, (e, f, s, ae, av) = run(m, atoms, gpus)
    n = len(atoms)
    pair = float(m.scale_shift.scale) * taps["e_pair"].abs() if "e_pair" in taps else torch.zeros(n, dtype=torch.float64)
    te = 1e-4 + (1e-5 * pair.sum().item() / n if rel else 0.0)
    tf = 1e-3 + (1e-5 * F.abs().max().item() if rel else 0.0)
    teps = 1e-4 + (1e-5 * pair.max().item() if rel else 0.0)
    de, df, ds = abs(e - E.item()) / n, np.abs(f - F.numpy()).max(), np.abs(s - S.numpy()).max()
    da = np.abs(ae - eps.numpy()).max()
    print(f"n={n} dE/atom={de:.2e} dF={df:.2e} dS={ds:.2e} deps={da:.2e} |F|max={F.abs().max():.3f} "
          f"|E_pair|={pair.sum().item():.3f}")
    assert de < te and df < tf and da < teps, (de, df, da, te, tf, teps)
    if all(atoms.get_pbc()):
        assert ds < 1e-3 + (1e-5 * np.abs(S.numpy()).max() if rel else 0.0), ds
    if virials:
        w = atomic_virials_ref(m, atoms).numpy()
        assert np.abs(av - w).max() < 1e-4 * max(1.0, np.abs(w).max()), np.abs(av - w).max()
        assert abs(ae.sum() - e) < 1e-6 * max(1.0, abs(e))
        if all(atoms.get_pbc()):
            np.testing.assert_allclose(av.sum(axis=0), s * atoms.get_volume() / 160.21766208,
                                       atol=2e-4 * max(1.0, np.abs(w).max()))
    return e, f, s, ae, av


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_diamond_mixed(opt, shape):
    check(model(opt, eq=SHAPES[shape], seed=1), diamond64(), virials=True)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_close_contact(opt, shape):
    check(model(opt, eq=SHAPES[shape], seed=2), close_contact(), rel=True, virials=True)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_cluster(opt, shape):
    check(model(opt, eq=SHAPES[shape], seed=3), cluster())


@pytest.mark.parametrize("shape", list(SHAPES))
def test_dimer_scan(shape):
    """the pair term alone (a ZBL-only model) from 0.5 A, where it dominates, to 3 A, past every ZBL cutoff here"""
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    m = model("zbl", eq=SHAPES[shape], seed=4)
    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode([0])
    for pair in (("Si", "Fe"), ("H", "O"), ("Fe", "Fe")):
        for r in np.linspace(0.5, 3.0, 11):
            a = dimer(r, *pair)
            E, F, _, eps = potential_ref(m, a, calc_stresses=False)
            e, f, _, ae, _ = d.evaluate(a, atomic=True)
            tf = 1e-3 + 1e-5 * F.abs().max().item()
            te = 1e-4 + 1e-5 * abs(E.item())
            assert abs(e - E.item()) / 2 < te and np.abs(f - F.numpy()).max() < tf, (pair, r, e, E.item())
            assert np.abs(ae - eps.numpy()).max() < 2 * te


@pytest.mark.parametrize("shape", list(SHAPES))
def test_large_cell_loops(shape):
    # 4096 atoms: every per-atom and per-edge grid covers the 132 SMs several times
    check(model("both", eq=SHAPES[shape], seed=5), mixed(si_diamond(8, seed=5)))


def test_89_elements_five_used():
    zs = tuple(range(1, 90))  # the MP-style element tables
    m = model("both", atomic_numbers=zs, seed=6)
    syms = ("H", "O", "Si", "Fe", "Cu")
    check(m, mixed(si_diamond(2, seed=6), seed=6, syms=syms), virials=True)


@pytest.mark.parametrize("parts", [2, 3])
def test_group_partitions_equal_one(parts):
    m = model("both", eq=True, seed=7, num_interactions=3)
    atoms = mixed(si_diamond(3, nz=10, seed=6))  # pair edges cross the slab walls
    _, (e1, f1, s1, a1, v1) = run(m, atoms)
    _, (e2, f2, s2, a2, v2) = run(m, atoms, gpus=[0] * parts)
    assert abs(e1 - e2) / len(atoms) < 1e-6
    assert np.abs(f1 - f2).max() < 1e-5 and np.abs(s1 - s2).max() < 1e-5
    assert np.abs(a1 - a2).max() < 1e-5 and np.abs(v1 - v2).max() < 1e-5


def test_eb_tap_is_the_transformed_basis():
    from scipy.spatial import cKDTree

    from oracle.graph_ref import neighbor_list

    m = model("both", seed=8)
    atoms = diamond64()
    taps = {}
    potential_ref(m, atoms, calc_forces=False, taps=taps)
    d, _ = run(m, atoms)
    ev, eb = d._engine.debug_tensor("e_vec"), d._engine.debug_tensor("eb")
    i1, i2, off, _, _ = neighbor_list(atoms.get_positions(), np.array(atoms.get_cell()), atoms.get_pbc().astype(np.int64),
                                      6.0, 0.0)
    pos = atoms.get_positions()
    vec = pos[i2] + off @ np.array(atoms.get_cell()) - pos[i1]
    dist, idx = cKDTree(vec).query(ev[:, :3].astype(np.float64))
    assert len(ev) == len(vec) and dist.max() < 1e-4 and len(set(idx.tolist())) == len(idx)
    ref = taps["eb"].numpy()[idx]
    assert np.abs(eb[:, :ref.shape[1]] - ref).max() < 1e-5 * max(1.0, np.abs(ref).max())


def test_zbl_term_is_not_silently_dropped_and_launch_counts():
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    atoms = close_contact()
    out, launches = {}, {}
    for opt in (None, "zbl", "agnesi"):
        dm = ScaleShiftMACE_Dist.from_existing(model(opt, seed=9))
        dm.enable_distributed_mode([0])
        out[opt] = dm.evaluate(atoms)
        launches[opt] = dm._engine.counts()["launches"]
    n = len(atoms)
    assert abs(out["zbl"][0] - out[None][0]) / n > 100 * 1e-4
    assert np.abs(out["zbl"][1] - out[None][1]).max() > 100 * 1e-3
    assert launches["zbl"] == launches[None] + 1 and launches["agnesi"] == launches[None], launches


def test_engine_refuses_malformed_keys():
    from distmlip_b200 import _lib
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(model("both", seed=10))
    desc = d._describe()
    cases = [
        ("pair_repulsion_fn.a_exp", None, "pair_repulsion_fn.a_exp"),                 # partial key set
        ("pair_repulsion_fn.c", torch.ones(3), "pair_repulsion_fn.c"),                # shape
        ("pair_repulsion_fn.p", torch.tensor(5.5), "integer"),                        # non-integer p
        ("pair_repulsion_fn.covalent_radii", torch.ones(20), "beyond"),               # Fe (26) beyond the table
        ("radial_embedding.distance_transform.covalent_radii", torch.ones(9), "beyond"),
        ("radial_embedding.distance_transform.a", None, "distance_transform.a"),
        ("pair_repulsion_fn.r_max", torch.tensor(6.0), "not used"),                   # a stray key
    ]
    for key, val, match in cases:
        sd = dict(d._state_dict)
        if val is None:
            sd.pop(key)
        else:
            sd[key] = val.float()
        eng = _lib.Engine(n_elem=desc.n_elem, n_blocks=desc.num_interactions, cutoff=desc.r_max, mace=desc, device=0)
        eng.load_state_dict(sd)
        with pytest.raises(Exception, match=match):
            eng.finalize()
        eng.close()


def test_calculator_committee_plain_and_zbl_agnesi():
    from distmlip_b200.implementations.mace import MACECalculator_Dist

    class Calc:  # the attribute surface of mace's MACECalculator
        def __init__(self, models):
            self.models, self.r_max = models, 6.0
            self.energy_units_to_eV, self.length_units_to_A = 1.0, 1.0

    ms = [model(None, seed=11), model("both", eq=True, seed=12)]
    atoms = close_contact()
    n = len(atoms)
    calc = MACECalculator_Dist.from_existing(Calc(ms))
    calc.enable_distributed_mode([0])
    calc.calculate(atoms)
    r = calc.results
    refs = [potential_ref(m, atoms) for m in ms]
    E = np.array([x[0].item() for x in refs])
    F = np.stack([x[1].numpy() for x in refs])
    S = np.stack([x[2].numpy() / 160.21766208 for x in refs])  # eV / A^3
    tf = 1e-3 + 1e-5 * np.abs(F).max()
    voigt = lambda t: np.array([t[0, 0], t[1, 1], t[2, 2], t[1, 2], t[0, 2], t[0, 1]])  # noqa: E731
    assert abs(r["energy"] - E.mean()) / n < 1e-4 + 1e-5 * np.abs(E).max() / n
    np.testing.assert_allclose(r["energies"], E, atol=1e-4 * n + 1e-5 * np.abs(E).max())
    np.testing.assert_allclose(r["forces_comm"], F, atol=tf)
    np.testing.assert_allclose(r["forces"], F.mean(0), atol=tf)
    np.testing.assert_allclose(r["stress"], voigt(S.mean(0)), atol=1e-5 + 1e-5 * np.abs(S).max())
    e0 = ms[0].atomic_energies_fn.atomic_energies.numpy()
    z_index = [ms[0].atomic_numbers.tolist().index(z) for z in atoms.get_atomic_numbers()]
    node = np.mean([x[3].numpy() for x in refs], axis=0) - e0[z_index]
    np.testing.assert_allclose(r["node_energy"], node, atol=1e-4 + 1e-5 * np.abs(node).max())
    assert Z_OF["Fe"] in atoms.get_atomic_numbers()
