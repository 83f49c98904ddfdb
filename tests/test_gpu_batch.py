"""GPU: batched evaluation (b2m_set_structures / b2m_compute_batch, DESIGN.md §12) of CHGNet, TensorNet and MACE.

One seeded batch B is used throughout: a perturbed 64-atom diamond, the 2-atom primitive Si cell (r_cut exceeds its
height: many images, reach > 1), a triclinic cell, a 300-atom rough cell, a slab (pbc 1, 1, 0), a cluster in a 40 A box
(pbc 0, 0, 0), structures of 7, 13 and 61 atoms (warps and 64-row tiles straddle structure boundaries) and two identical
copies of one structure, with mixed species.

The graph of a batch is the disjoint union of the structures' graphs, in each structure's own order; every result of a
structure in a batch equals a single evaluation of it to fp32 round-off.  The fp32 atomics and the tile-wise scatters add
in another order when tiles straddle structures, so the tolerances are those the other tests allow between two
evaluations of one structure, with an fp32 floor on the energy: energy 1e-8 relative or 5e-8 eV per atom (observed on an
H100: 1.5e-8 eV per atom for CHGNet's 2-atom cell; TensorNet and MACE energies bit-identical), forces 1e-8 relative or
5e-8 eV/A for CHGNet and TensorNet (tests/test_gpu_atomic.py) and 1e-6 eV/A for MACE (tests/test_gpu_mace*.py allow
1e-5 between partition layouts; observed 1.5e-7), stress 1e-5 relative + 1e-6 GPa (the sum rule of the per-atom
virials, through which a batch's stress comes), per-atom values to tests/test_gpu_atomic.py's bounds.
"""
import numpy as np
import pytest
import torch

from distmlip_b200.structures import Z_OF, SimpleAtoms, rough_cell, si_diamond
from tests._util import engine_from_model, key5, make_model, oracle_graph
from tests.test_gpu_tensornet import tn_engine
from tests.test_oracle_tensornet import make_tn

pytestmark = pytest.mark.gpu
B2M_ERR_INVALID, B2M_ERR_STATE = -1, -6
TOL_EPS = 2e-6                                 # eV, per-atom energies (tests/test_gpu_atomic.py)
TOL_W = 4e-5                                   # per-atom virials over max |w| (the CHGNet bound there; TensorNet 2e-5)
SCALING = dict(data_mean=0.7, data_std=1.3)


def mixed(atoms, other="O", every=3, pbc=None):
    sym = [other if i % every == 0 else s for i, s in enumerate(atoms.get_chemical_symbols())]
    return SimpleAtoms(sym, atoms.get_positions(), np.array(atoms.get_cell()),
                       pbc=atoms.get_pbc() if pbc is None else pbc)


def triclinic(n, seed):
    a = rough_cell(n, seed=seed)
    frac = a.get_positions() @ np.linalg.inv(np.array(a.get_cell()))
    L = np.array(a.get_cell())[0, 0]
    cell = L * np.array([[1.0, 0.0, 0.0], [0.25, 1.05, 0.0], [0.15, -0.2, 1.1]])
    return SimpleAtoms(["Si"] * n, frac @ cell, cell)


def batch_B():
    prim = SimpleAtoms(["Si", "Si"], np.array([[0.0, 0.0, 0.0], [1.36, 1.34, 1.37]]),
                       np.array([[0.0, 2.715, 2.715], [2.715, 0.0, 2.715], [2.715, 2.715, 0.0]]))
    slab = si_diamond(2, sigma=0.15, seed=5)
    c = rough_cell(20, seed=6)
    cluster = SimpleAtoms(["Si"] * 20, c.get_positions() + 15.0, np.eye(3) * 40.0, pbc=(False, False, False))
    twin = rough_cell(13, seed=9)
    return [mixed(si_diamond(2, sigma=0.15, seed=1)), mixed(prim, every=2), mixed(triclinic(13, seed=2)),
            mixed(rough_cell(300, seed=4), every=2), mixed(slab, pbc=(True, True, False)), mixed(cluster),
            mixed(rough_cell(7, seed=7)), mixed(rough_cell(13, seed=8), every=4), mixed(rough_cell(61, seed=10)),
            mixed(twin), mixed(twin)]


TWINS = (9, 10)


# ------------------------------------------------------------------ the model families
def mace_model(kind):
    kw = dict(C=32, r_max=6.0, scale=8.0, seed=1)
    if kind == "mace_0e":
        from oracle.mace_ref import make_mace
        return make_mace(**kw)
    if kind == "mace_0e1o":
        from tests.mace_eq_ref import make_mace_eq
        return make_mace_eq(**kw)
    if kind == "mace_0e1o2e":
        from tests.mace_l2_ref import make_mace_l2
        return make_mace_l2(**kw)
    from tests.test_oracle_mace_zbl import model
    return model("both")


class Family:
    """an engine of one model family, its species map and its float64 oracle"""

    def __init__(self, kind, device=0):
        self.kind = kind
        if kind == "chgnet":
            self.model = make_model(seed=2)
            refs = np.linspace(-0.5, 0.5, len(self.model.element_types))
            self.eng = engine_from_model(self.model, device=device, element_refs=refs, **SCALING)
            self.index = {s: i for i, s in enumerate(self.model.element_types)}
        elif kind == "tensornet":
            self.model = make_tn(seed=3, scale=1.5)
            refs = np.linspace(-0.5, 0.5, len(self.model.element_types))
            self.eng = tn_engine(self.model, device=device, element_refs=refs, **SCALING)
            self.index = {s: i for i, s in enumerate(self.model.element_types)}
        else:
            from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

            self.model = mace_model(kind)
            self.dist = ScaleShiftMACE_Dist.from_existing(self.model)
            self.dist.enable_distributed_mode(device if isinstance(device, list) else [device])
            self.eng = self.dist._engine
            zs = [int(z) for z in torch.as_tensor(self.model.atomic_numbers).tolist()]
            self.index = {s: zs.index(z) for s, z in Z_OF.items() if z in zs}

    def species(self, atoms):
        return np.array([self.index[s] for s in atoms.get_chemical_symbols()], dtype=np.int32)

    def set_structure(self, atoms):
        self.eng.set_structure(atoms.get_positions(), np.array(atoms.get_cell()), self.species(atoms),
                               np.asarray(atoms.get_pbc(), dtype=np.int32))

    def set_structures(self, atoms_list):
        self.eng.set_structures([len(a) for a in atoms_list], np.concatenate([a.get_positions() for a in atoms_list]),
                                np.array([np.array(a.get_cell()) for a in atoms_list]),
                                np.concatenate([self.species(a) for a in atoms_list]),
                                np.array([np.asarray(a.get_pbc(), dtype=np.int32) for a in atoms_list]))

    def oracle(self, atoms):
        """float64 (E, F, S) of one structure without the engine's scaling (use with a plain engine)"""
        if self.kind == "chgnet":
            from oracle.chgnet_ref import potential_ref
            E, F, S, _ = potential_ref(make_model(seed=2).double(), atoms, dtype=torch.float64)
            return E, F, S
        if self.kind == "tensornet":
            from tests.test_gpu_tensornet import oracle_efs
            (E, F, S), _og = oracle_efs(self.model, atoms)
            return E, F, S
        ref = {"mace_0e": "oracle.mace_ref", "mace_0e1o": "tests.mace_eq_ref", "mace_0e1o2e": "tests.mace_l2_ref",
               "mace_zbl_agnesi": "tests.mace_zbl_ref"}[self.kind]
        import importlib
        E, F, S, _eps = importlib.import_module(ref).potential_ref(self.model, atoms)
        return E, F, S


def singles(fam, atoms_list, site=False):
    """per structure: energy, forces, stress, per-atom energies, per-atom virials (, site-wise) of b2m_compute"""
    fam.eng.set_atomic(True)
    out = []
    for a in atoms_list:
        fam.set_structure(a)
        e, f, s = fam.eng.compute()
        ae, av = fam.eng.atomic()
        out.append((e, f, s, ae, av) + ((fam.eng.sitewise(),) if site else ()))
    return out


def batched(fam, atoms_list, site=False):
    fam.set_structures(atoms_list)
    E, F, S = fam.eng.compute_batch()
    AE, AV = fam.eng.atomic()
    SW = fam.eng.sitewise() if site else None
    cut = np.cumsum([len(a) for a in atoms_list])[:-1]
    parts = zip(np.split(F, cut), np.split(AE, cut), np.split(AV, cut),
                np.split(SW, cut) if site else [None] * len(atoms_list))
    return [(E[k], f, S[k], ae, av) + ((sw,) if site else ()) for k, (f, ae, av, sw) in enumerate(parts)]


def tol_e(e0, n):
    return max(1e-8 * abs(e0), 5e-8 * n)


def tol_f(f0, floor=5e-8):
    return max(1e-8 * float(np.abs(f0).max()), floor)


def force_floor(kind):
    return 1e-6 if kind.startswith("mace") else 5e-8


def assert_same(got, want, what, ffloor=5e-8):
    e, f, s, ae, av = got[:5]
    e0, f0, s0, ae0, av0 = want[:5]
    ftol = tol_f(f0, ffloor)
    de, df, ds = abs(e - e0), np.abs(f - f0).max(), np.abs(s - s0).max()
    deps, dw = np.abs(ae - ae0).max(), np.abs(av - av0).max() / max(np.abs(av0).max(), 1e-30)
    print(f"{what}: |dE| {de:.2e} |dF| {df:.2e} |dS| {ds:.2e} |deps| {deps:.2e} |dw|/max|w| {dw:.2e}")
    assert de <= tol_e(e0, len(f0)), (what, e, e0)
    assert df <= ftol, (what, df, ftol)
    assert ds <= 1e-5 * np.abs(s0).max() + 1e-6, (what, s, s0)
    assert deps <= TOL_EPS, (what, deps)
    assert dw <= TOL_W, (what, dw)
    if len(want) > 5:
        assert np.abs(got[5] - want[5]).max() <= 1e-6, (what, np.abs(got[5] - want[5]).max())


FAMILIES = ["chgnet", "tensornet", "mace_0e", "mace_0e1o", "mace_0e1o2e", "mace_zbl_agnesi"]


@pytest.fixture(scope="module")
def B():
    return batch_B()


# ------------------------------------------------------------------ 1. graph
def test_graph_is_the_disjoint_union_of_the_single_graphs(B):
    fam = Family("chgnet")
    fam.set_structures(B)
    c = fam.eng.counts()
    edges, bonds, angles = (fam.eng.partition_info(k) for k in (3, 4, 5))
    assert c["n_own"] == sum(len(a) for a in B) and c["n_halo"] == 0 and c["world"] == 1
    off = np.r_[0, np.cumsum([len(a) for a in B])]
    for k, a in enumerate(B):
        lo, hi = off[k], off[k + 1]
        mine = (edges[:, 1] >= lo) & (edges[:, 1] < hi)
        bmine = (bonds[:, 1] >= lo) & (bonds[:, 1] < hi)
        amine = (angles[:, 2] >= lo) & (angles[:, 2] < hi)
        e_b = edges[mine] - [lo, lo, 0, 0, 0]
        b_b = bonds[bmine] - [lo, lo, 0, 0, 0]
        a_b = [(tuple(bonds[i]), tuple(bonds[o]), int(ce) - lo) for i, o, ce in angles[amine]]
        assert ((e_b[:, 0] >= 0) & (e_b[:, 0] < len(a))).all() and ((b_b[:, 0] >= 0) & (b_b[:, 0] < len(a))).all()
        fam.set_structure(a)
        e_s, b_s, an_s = (fam.eng.partition_info(w) for w in (3, 4, 5))
        np.testing.assert_array_equal(e_b, e_s)  # same rows, same edge order
        np.testing.assert_array_equal(b_b, b_s)
        a_s = [(tuple(b_s[i] + [lo, lo, 0, 0, 0]), tuple(b_s[o] + [lo, lo, 0, 0, 0]), int(ce)) for i, o, ce in an_s]
        assert a_b == a_s
        og = oracle_graph(a, rc=fam.model.cutoff, rb=fam.model.three_body_cutoff)
        assert sorted(key5(e_b)) == sorted(key5(np.column_stack([og["i1"], og["i2"], og["off"]])))
        be = og["bond_edges"]
        assert sorted(key5(b_b)) == sorted(key5(np.column_stack([og["i1"][be], og["i2"][be], og["off"][be]])))
        assert len(a_b) == len(og["la"])
        print(f"structure {k}: {len(a)} atoms, {len(e_b)} edges, {len(b_b)} bonds, {len(a_b)} angles")
    fam.eng.close()


# ------------------------------------------------------------------ 2. batch equals single
@pytest.mark.parametrize("kind", FAMILIES)
def test_batch_equals_single_calls(B, kind):
    fam = Family(kind)
    site = kind == "chgnet"
    want = singles(fam, B, site)
    got = batched(fam, B, site)
    for k in range(len(B)):
        assert_same(got[k], want[k], f"{kind} structure {k}", force_floor(kind))
    fam.eng.close()


# ------------------------------------------------------------------ 3. batch against the float64 oracle
@pytest.mark.parametrize("kind", FAMILIES)
def test_batch_matches_the_float64_oracle(B, kind):
    fam = Family(kind)
    if kind in ("chgnet", "tensornet"):  # the oracle has no scaling: a plain engine
        fam.eng.close()
        fam.eng = (engine_from_model if kind == "chgnet" else tn_engine)(fam.model)
    pick = [0, 1, 2, 5]
    atoms = [B[k] for k in pick]
    fam.set_structures(atoms)
    E, F, S = fam.eng.compute_batch()
    cut = np.cumsum([len(a) for a in atoms])[:-1]
    for a, e, f, s in zip(atoms, E, np.split(F, cut), S):
        Eo, Fo, So = fam.oracle(a)
        n = len(a)
        de, df = abs(e - float(Eo)) / n, np.abs(f - Fo.numpy()).max()
        ds = np.abs(s - So.numpy()).max() if all(a.get_pbc()) else 0.0
        print(f"{kind} n={n}: dE/atom {de:.2e} dF {df:.2e} dS {ds:.2e}")
        assert de < 1e-4 and df < 1e-3 and ds < 1e-3, (de, df, ds)
    fam.eng.close()


# ------------------------------------------------------------------ 4. symmetries
@pytest.mark.parametrize("kind", ["chgnet", "mace_0e1o"])
def test_order_singleton_twins_and_return_to_single(B, kind):
    fam = Family(kind)
    fam.eng.set_atomic(True)
    fam.set_structure(B[3])
    before = fam.eng.compute()
    fwd = batched(fam, B)
    rev = batched(fam, B[::-1])
    for k in range(len(B)):
        assert_same(rev[len(B) - 1 - k], fwd[k], f"{kind} reversed, structure {k}", force_floor(kind))
    assert_same(fwd[TWINS[1]], fwd[TWINS[0]], f"{kind} twins", force_floor(kind))
    one = batched(fam, [B[2]])[0]
    assert_same(one, singles(fam, [B[2]])[0], f"{kind} batch of one", force_floor(kind))
    fam.set_structure(B[3])
    after = fam.eng.compute()
    assert abs(after[0] - before[0]) <= tol_e(before[0], len(before[1]))
    assert np.abs(after[1] - before[1]).max() <= tol_f(before[1], force_floor(kind))
    assert np.abs(after[2] - before[2]).max() <= 1e-6 * np.abs(before[2]).max() + 1e-7
    fam.eng.close()


# ------------------------------------------------------------------ 5. scale
def test_1500_structures_in_one_pass():
    rng = np.random.default_rng(21)
    atoms = []
    for k in range(1500):
        a = si_diamond(1, sigma=0.1, seed=100 + k, nz=int(rng.integers(1, 9)))  # 8 .. 64 atoms
        atoms.append(mixed(a, every=int(rng.integers(2, 5))))
    fam = Family("chgnet")
    fam.set_structures(atoms[:1])
    fam.eng.compute_batch()
    launches_1 = fam.eng.counts()["launches"]
    got = batched(fam, atoms)
    c = fam.eng.counts()
    print(f"{len(atoms)} structures, {c['n_own']} atoms, {c['n_edges']} edges, {c['n_angles']} angles, "
          f"{c['launches']} launches (S = 1: {launches_1}), timings {fam.eng.timings()}")
    assert c["launches"] == launches_1  # the batch is one pass, not a loop
    pick = rng.choice(len(atoms), 20, replace=False)
    want = singles(fam, [atoms[k] for k in pick])
    for k, w in zip(pick, want):
        assert_same(got[k], w, f"structure {k} of 1500")
    fam.eng.close()


# ------------------------------------------------------------------ 6. refusals
def expect(code, text, fn, *args, **kw):
    from distmlip_b200._lib import B2MError

    with pytest.raises(B2MError) as ei:
        fn(*args, **kw)
    assert ei.value.code == code and text in str(ei.value), str(ei.value)


def test_refusals_and_what_works_while_a_batch_is_resident(B):
    fam = Family("chgnet")
    eng = fam.eng
    small = B[6:9]
    n = [len(a) for a in small]
    cart = np.concatenate([a.get_positions() for a in small])
    cells = np.array([np.array(a.get_cell()) for a in small])
    sp = np.concatenate([fam.species(a) for a in small])
    pbc = np.ones((3, 3), dtype=np.int32)
    expect(B2M_ERR_INVALID, "at least one structure", eng.set_structures, [], np.zeros((0, 3)), np.zeros((0, 3, 3)),
           np.zeros(0), np.zeros((0, 3)))
    expect(B2M_ERR_INVALID, "structure 1: no atoms", eng.set_structures, [n[0], 0, n[1] + n[2]], cart, cells, sp, pbc)
    bad = pbc.copy()
    bad[1, 2] = 2
    expect(B2M_ERR_INVALID, "structure 1: pbc flags", eng.set_structures, n, cart, cells, sp, bad)
    sing = cells.copy()
    sing[2, 2] = sing[2, 1]
    expect(B2M_ERR_INVALID, "structure 2: singular lattice", eng.set_structures, n, cart, sing, sp, pbc)
    lone = SimpleAtoms(["Si"], np.array([[20.0, 20.0, 20.0]]), np.eye(3) * 40.0, pbc=(False, False, False))
    expect(B2M_ERR_INVALID, "structure 1 has no edges", fam.set_structures, [small[0], lone, small[1]])
    eng.set_heat_flux(20.0)
    expect(B2M_ERR_STATE, "heat flux", eng.set_structures, n, cart, cells, sp, pbc)
    eng.set_heat_flux(0.0)
    eng.set_partition(0, 2)
    expect(B2M_ERR_INVALID, "one partition", eng.set_structures, n, cart, cells, sp, pbc)
    eng.set_partition(0, 1)
    fam.set_structure(small[0])
    expect(B2M_ERR_STATE, "no batch is resident", eng.compute_batch)
    # resident batch: the single-structure calls refuse, the inspection calls work
    eng.set_atomic(False)
    eng.set_structures(n, cart, cells, sp, pbc)
    E, F, S = eng.compute_batch(forces=False, stress=False)
    assert F is None and S is None and E.shape == (3,)
    ae, _ = eng.atomic(virials=False)
    assert ae.shape == (sum(n),)
    expect(B2M_ERR_STATE, "virials", eng.atomic)
    for call in (eng.compute, eng.results, lambda: eng.compute_resident(1),
                 lambda: eng.compute_heat_flux(np.zeros((sum(n), 3)))):
        expect(B2M_ERR_STATE, "a batch is resident", call)
    E, F, S = eng.compute_batch()
    assert eng.atomic()[1].shape == (sum(n), 3, 3) and eng.sitewise().shape == (sum(n),)
    assert eng.counts()["n_own"] == sum(n) and len(eng.partition_info(0)) == sum(n)
    assert eng.timings()["graph_ms"] > 0
    eng.release_workspace()
    eng.set_structures(n, cart, cells, sp, pbc)
    E2, F2, S2 = eng.compute_batch()
    assert all(abs(E2[k] - E[k]) <= tol_e(E[k], n[k]) for k in range(3)) and np.abs(F2 - F).max() <= tol_f(F)
    eng.close()
    group = Family("chgnet", device=[0, 0])
    expect(B2M_ERR_INVALID, "one partition", group.set_structures, small)
    group.eng.close()


def test_python_entry_points_refuse_a_group():
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    dm = CHGNet_Dist.from_existing(make_model(seed=2))
    dm.enable_distributed_mode([0, 0])
    with pytest.raises(NotImplementedError, match="one GPU and one partition"):
        Potential_Dist(model=dm).forward_batch(batch_B()[6:8])
    with pytest.raises(NotImplementedError, match="heat flux"):
        Potential_Dist(model=dm, calc_heat_flux=True).forward_batch(batch_B()[6:8])
    dm._engine.close()


def test_forward_batch_equals_forward(B):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist

    model = make_model(seed=2)
    dm = CHGNet_Dist.from_existing(model)
    dm.enable_distributed_mode([0])
    pot = Potential_Dist(model=dm, calc_site_wise=True, calc_atomic=True, **SCALING)
    got = pot.forward_batch(B)
    ae_b = pot.atomic_energies
    for k, a in enumerate(B):
        E, F, S, _h, site = pot(a)
        Eb, Fb, Sb, _hb, siteb = got[k]
        assert abs(float(Eb) - float(E)) <= tol_e(float(E), len(a))
        assert float((Fb - F).abs().max()) <= tol_f(F.numpy())
        assert float((Sb - S).abs().max()) <= 1e-5 * float(S.abs().max()) + 1e-6
        assert float((siteb - site).abs().max()) <= 1e-6
        assert float((ae_b[k] - pot.atomic_energies).abs().max()) <= TOL_EPS
    dm._engine.close()
