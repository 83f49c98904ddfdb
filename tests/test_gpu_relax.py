"""GPU: batched relaxation (b2m_relax_batch, DESIGN.md §13) against the host loop.

The host loop is tests/relax_ref.py's float64 FIRE (+ Frechet cell filter) driven by b2m_compute_batch of the same
engine, with the strain derivative W summed in f64 from the per-atom virials as the device sums it: the only
difference is where FIRE runs.  Two evaluations of one geometry agree to fp32 round-off (the fp32 atomics add in
another order), and a structure's results in a batch equal its results alone to §12's batch tolerances, so the two
loops agree to: positions 1e-6 A, cells 1e-8 relative, energies 1e-6 eV per atom, and identical step counts and
converged flags when no FIRE branch or convergence test along the way is marginal (asserted).
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy.linalg import expm

from distmlip_b200 import _lib
from distmlip_b200.structures import SimpleAtoms, rough_cell, si_diamond
from tests.relax_ref import FIRE_DEFAULTS, Fire, relax
from tests.test_gpu_batch import Family, batch_B, mixed, triclinic

pytestmark = pytest.mark.gpu
B2M_ERR_INVALID, B2M_ERR_STATE = -1, -6
TOL_X, TOL_CELL, TOL_E = 1e-6, 1e-8, 1e-6
MARGIN = 1e-6


def inputs(fam, atoms_list):
    return ([len(a) for a in atoms_list], np.concatenate([a.get_positions() for a in atoms_list]),
            np.array([np.array(a.get_cell()) for a in atoms_list]),
            np.concatenate([fam.species(a) for a in atoms_list]),
            np.array([np.asarray(a.get_pbc(), dtype=np.int32) for a in atoms_list]))


def host_loop(fam, atoms_list, fmax, steps, relax_cell, p=0.0):
    def evaluate(ids, geos):
        subset = [SimpleAtoms(atoms_list[s].get_chemical_symbols(), x, c, pbc=atoms_list[s].get_pbc())
                  for s, (x, c) in zip(ids, geos)]
        fam.eng.set_structures(*inputs(fam, subset))
        e, f, _ = fam.eng.compute_batch()
        _, w = fam.eng.atomic(virials=True)
        cut = np.cumsum([len(a) for a in subset])[:-1]
        return [(ek, fk, wk.astype(np.float64).sum(axis=0)) for ek, fk, wk in zip(e, np.split(f, cut), np.split(w, cut))]

    return relax([(a.get_positions(), np.array(a.get_cell())) for a in atoms_list], evaluate, fmax, steps, relax_cell,
                 p=p)


def device(fam, atoms_list, **kw):
    return fam.eng.relax_batch(*inputs(fam, atoms_list), **kw)


def compare(atoms_list, dev, host, fmax):
    cut = np.cumsum([len(a) for a in atoms_list])[:-1]
    for k, (a, x, h) in enumerate(zip(atoms_list, np.split(dev["cart"], cut), host)):
        assert dev["steps"][k] == h["steps"] and dev["converged"][k] == h["converged"], k
        assert min(h["margins"], default=1.0) > MARGIN, (k, min(h["margins"]))
        assert all(abs(fm - fmax) > 1e-4 * max(fmax, 1e-30) for fm in h["fmaxes"]), k  # no marginal convergence test
        np.testing.assert_allclose(x, h["positions"], atol=TOL_X, err_msg=f"structure {k}")
        np.testing.assert_allclose(dev["lattices"][k], h["cell"], rtol=TOL_CELL, atol=TOL_CELL * np.abs(h["cell"]).max())
        tr = dev["trace"][k]
        n_ev = h["steps"] + 1
        np.testing.assert_allclose(tr[:n_ev], h["energies"], rtol=0, atol=TOL_E * len(a), err_msg=f"structure {k}")
        assert np.isnan(tr[n_ev:]).all()
        np.testing.assert_allclose(dev["energies"][k], h["energy"], rtol=0, atol=TOL_E * len(a))


def periodic_pair():
    return [mixed(si_diamond(2, sigma=0.15, seed=1)), mixed(triclinic(13, seed=2))]


@pytest.mark.parametrize("kind", ["chgnet", "tensornet", "mace_0e", "mace_0e1o2e"])
@pytest.mark.parametrize("relax_cell,p", [(False, 0.0), (True, 0.002)])
def test_device_loop_equals_host_loop(kind, relax_cell, p):
    fam = Family(kind)
    atoms = periodic_pair()
    host = host_loop(fam, atoms, 0.0, 30, relax_cell, p)
    dev = device(fam, atoms, fmax=0.0, steps=30, relax_cell=relax_cell, scalar_pressure=p)
    compare(atoms, dev, host, 0.0)
    assert not dev["converged"].any() and (dev["steps"] == 30).all()


def pick_fmax(host):
    """an fmax, from the trajectories of a run that never converges, at the middle of a gap between the max-row forces
    they visit (so no convergence test is marginal), chosen so that at least one structure runs out of steps and the
    others converge at as many different steps as possible"""
    vals = np.unique(np.concatenate([h["fmaxes"] for h in host]))
    best, best_key = None, None
    for lo, hi in zip(vals[:-1], vals[1:]):
        if hi - lo < 2e-3 * hi:
            continue
        f = 0.5 * (lo + hi)
        first = [next((t for t, fm in enumerate(h["fmaxes"]) if fm < f), None) for h in host]
        stops = [t for t in first if t is not None]
        if len(stops) == len(first) or not stops:
            continue
        key = (len(set(stops)), hi - lo)
        if best_key is None or key > best_key:
            best, best_key = f, key
    assert best is not None
    return best


@pytest.mark.parametrize("kind", ["chgnet", "tensornet", "mace_0e"])
@pytest.mark.parametrize("relax_cell,p", [(False, 0.0), (True, 0.0), (True, 0.003)])
def test_mixed_batch_compacts_and_matches_each_structure_alone(kind, relax_cell, p):
    fam = Family(kind)
    B = batch_B()
    atoms = [a for a in B if np.asarray(a.get_pbc()).all()] if relax_cell else B
    steps = 20
    probe = host_loop(fam, atoms, 0.0, steps, relax_cell, p)
    fmax = pick_fmax(probe)
    host = host_loop(fam, atoms, fmax, steps, relax_cell, p)
    dev = device(fam, atoms, fmax=fmax, steps=steps, relax_cell=relax_cell, scalar_pressure=p)
    compare(atoms, dev, host, fmax)
    assert dev["converged"].any() and not dev["converged"].all()
    assert len(set(dev["steps"][dev["converged"]].tolist())) > 1
    # each structure alone in a batch of one
    cut = np.cumsum([len(a) for a in atoms])[:-1]
    for k, a in enumerate(atoms):
        one = device(fam, [a], fmax=fmax, steps=steps, relax_cell=relax_cell, scalar_pressure=p)
        assert one["steps"][0] == dev["steps"][k] and one["converged"][0] == dev["converged"][k]
        np.testing.assert_allclose(np.split(dev["cart"], cut)[k], one["cart"], atol=TOL_X)
        np.testing.assert_allclose(dev["lattices"][k], one["lattices"][0], rtol=TOL_CELL,
                                   atol=TOL_CELL * np.abs(one["lattices"][0]).max())
        np.testing.assert_allclose(dev["trace"][k], one["trace"][0], rtol=0, atol=TOL_E * len(a))
    # the results are those of a fresh evaluation of the returned geometries
    final = [SimpleAtoms(a.get_chemical_symbols(), x, c, pbc=a.get_pbc())
             for a, x, c in zip(atoms, np.split(dev["cart"], cut), dev["lattices"])]
    fam.set_structures(final)
    e, f, s = fam.eng.compute_batch()
    np.testing.assert_allclose(dev["energies"], e, rtol=1e-8, atol=5e-8 * max(len(a) for a in atoms))
    np.testing.assert_allclose(dev["forces"], f, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(dev["stress"], s, rtol=1e-5, atol=1e-5)


def test_launches_per_step_do_not_depend_on_the_batch():
    fam = Family("chgnet")
    a = mixed(rough_cell(7, seed=7))
    device(fam, [a], fmax=0.0, steps=2)
    one = fam.eng.counts()["launches"]
    device(fam, [a] * 500, fmax=0.0, steps=2)
    assert fam.eng.counts()["launches"] == one


def test_python_surface_on_the_engine():
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist
    from oracle.mace_ref import make_mace

    model = ScaleShiftMACE_Dist.from_existing(make_mace(C=32, r_max=6.0, scale=8.0, seed=1))
    model.enable_distributed_mode([0])
    atoms = periodic_pair()
    before = [a.get_positions().copy() for a in atoms]
    out = model.relax_batch(atoms, fmax=0.0, steps=5, relax_cell=True, scalar_pressure=0.001, maxstep=0.1)
    for a, x, o in zip(atoms, before, out):
        np.testing.assert_array_equal(a.get_positions(), x)
        assert o["steps"] == 5 and not o["converged"] and len(o["energies"]) == 6
        e, f, s, _, _ = model.evaluate(o["final_structure"])
        np.testing.assert_allclose(o["energy"], e, rtol=1e-7)
        np.testing.assert_allclose(o["stress"], s / 160.21766208, rtol=1e-4, atol=1e-7)


def test_c_refusals():
    fam = Family("chgnet")
    B = batch_B()
    ok = [B[0]]

    def refused(code, match, atoms_list=ok, **kw):
        with pytest.raises(_lib.B2MError, match=match) as ei:
            device(fam, atoms_list, **kw)
        assert ei.value.code == code

    refused(B2M_ERR_INVALID, "structure 1: relax_cell needs a periodic", [B[0], B[4]], relax_cell=True)
    refused(B2M_ERR_INVALID, "steps must be >= 0", steps=-1)
    refused(B2M_ERR_INVALID, "finite", dt=float("nan"))
    refused(B2M_ERR_INVALID, "finite", scalar_pressure=float("inf"))
    for k in ("dt", "maxstep", "dtmax"):
        refused(B2M_ERR_INVALID, "must be > 0", **{k: 0.0})
    lone = SimpleAtoms(["Si"], np.zeros((1, 3)) + 5.0, np.eye(3) * 30.0, pbc=(False, False, False))
    refused(B2M_ERR_INVALID, "relaxation step 0: structure 2 has no edges", [B[0], B[1], lone], relax_cell=False)
    with pytest.raises(_lib.B2MError) as ei:
        fam.eng.relax_batch([], np.zeros((0, 3)), np.zeros((0, 3, 3)), np.zeros(0, np.int32), np.zeros((0, 3)))
    assert ei.value.code == B2M_ERR_INVALID
    # the handle stays usable
    r = device(fam, ok, fmax=0.0, steps=1)
    assert r["steps"][0] == 1
    fam.eng.set_heat_flux(8.0)
    refused(B2M_ERR_STATE, "heat flux")


# ------------------------------------------------------------------------------------------ one step, kernel level
def build_relax_shim(outdir):
    """Compile tests/relax_shim.cu against the built libb200mlip.so into outdir (as kernel_units_ref.build_shim)."""
    from distmlip_b200 import build

    lib = build.build()
    libdir = os.path.dirname(lib)
    here = os.path.dirname(os.path.abspath(__file__))
    out = os.path.join(str(outdir), "librelax_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + [
        "-I", build.CSRC, "-I", os.path.join(here, "..", "include"), "-shared", os.path.join(here, "relax_shim.cu"),
        "-o", out, "-L", libdir, "-l:" + os.path.basename(lib), "-Xlinker", "-rpath," + libdir]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def relax_shim(tmp_path_factory):
    return build_relax_shim(tmp_path_factory.mktemp("relax_shim"))


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# natoms, force scale (eV/A), virial scale (eV): one structure larger than a block, virials up to 1e3 eV, and one
# structure with forces far below fmax
SHAPES = [(1, 1.0, 1.0), (5, 0.5, 100.0), (37, 2.0, 1000.0), (300, 1.0, 300.0), (8, 1e-7, 1e-7)]


@pytest.mark.parametrize("it,steps", [(0, 10), (3, 10), (3, 3)])
@pytest.mark.parametrize("relax_cell,p", [(False, 0.0), (True, 0.0), (True, 0.01)])
def test_one_step_equals_relax_ref(relax_shim, it, steps, relax_cell, p):
    rng = np.random.default_rng(17 + it + 7 * relax_cell + int(1000 * p))
    fmax, k, data_mean = 1e-3, 1.3, 0.4
    fire = dict(FIRE_DEFAULTS, dtmax=0.6)
    natoms = np.array([n for n, _, _ in SHAPES], dtype=np.int64)
    S, N = len(natoms), int(natoms.sum())
    cell0 = np.array([np.eye(3) * 10.0 + rng.normal(0, 0.8, (3, 3)) for _ in range(S)])
    X = np.array([n * 0.03 * rng.standard_normal((3, 3)) for n in natoms]) if relax_cell else np.zeros((S, 3, 3))
    F = np.array([expm(x / n) for x, n in zip(X, natoms)])
    r0 = rng.uniform(0, 10, (N, 3))
    v = rng.normal(0, 0.3, (N, 3)) if it else np.zeros((N, 3))
    vc = rng.normal(0, 0.3, (S, 3, 3)) if it and relax_cell else np.zeros((S, 3, 3))
    dt = rng.uniform(0.05, 0.5, S)
    a = rng.uniform(0.05, 0.2, S)
    nsteps = rng.integers(0, 11, S).astype(np.int32)
    cut = np.cumsum(natoms)[:-1]
    forces = np.concatenate([rng.normal(0, fs, (n, 3)) for n, fs, _ in SHAPES]).astype(np.float32)
    bsum = np.zeros((S, 10))
    bsum[:, 0] = rng.normal(0, 10, S)
    bsum[:, 1:] = np.array([rng.normal(0, ws, 9) for _, _, ws in SHAPES])
    # the reference step
    ref = []
    for s in range(S):
        o = Fire(r0[cut[s - 1] if s else 0:][:natoms[s]], cell0[s], relax_cell, k=k, p=p, **fire)
        o.X, o.dt, o.a, o.nsteps = X[s].copy(), dt[s], a[s], int(nsteps[s])
        vs = v[cut[s - 1] if s else 0:][:natoms[s]]
        o.v = (np.vstack([vs, vc[s]]) if relax_cell else vs.copy()) if it else None
        fs = forces[cut[s - 1] if s else 0:][:natoms[s]].astype(np.float64)
        g = o.forces(fs, bsum[s, 1:].reshape(3, 3))
        fm = float(np.sqrt((g ** 2).sum(1).max()))
        flag = 1 if fm < fmax else (2 if it >= steps else 0)
        if flag == 0:
            o.step(g)
            assert min(o.margins, default=1.0) > 1e-6
        ref.append((o, flag, fm))
    # the kernels
    d = lambda x: np.array(x, dtype=np.float64, order="C")  # noqa: E731  (copies: the shim writes into them)
    cfg = d([fmax, fire["maxstep"], fire["dtmax"], fire["Nmin"], fire["finc"], fire["fdec"], fire["astart"], fire["fa"],
             k, p])
    cell0_, X_, vc_, F_, dt_, a_, v_, r0_ = map(d, (cell0, X, vc, F, dt, a, v, r0))
    ns_ = nsteps.copy()
    stat = np.zeros((S, 12))
    res_f = np.zeros((N, 3), np.float32)
    res_e = np.zeros(S)
    res_s = np.zeros((S, 9))
    msg = ctypes.create_string_buffer(512)
    P = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = relax_shim.shim_relax_step(
        ctypes.c_int(S), P(natoms), ctypes.c_int(it), ctypes.c_int(steps), ctypes.c_int(int(relax_cell)), P(cfg),
        P(cell0_), P(X_), P(vc_), P(F_), P(dt_), P(a_), P(ns_), P(forces), P(d(bsum)), ctypes.c_double(data_mean),
        P(v_), P(r0_), P(stat), P(res_f), P(res_e), P(res_s), msg, ctypes.c_int(len(msg)))
    assert rc == 0, msg.value
    assert [f for _, f, _ in ref][:4] == [2 if it >= steps else 0] * 4  # the last may converge, the others do not
    for s, (o, flag, fm) in enumerate(ref):
        rows = slice(cut[s - 1] if s else 0, (cut[s - 1] if s else 0) + natoms[s])
        assert int(stat[s, 0]) == flag, s
        assert rel(stat[s, 1], bsum[s, 0] + data_mean) < 1e-15 and rel(stat[s, 2], fm) < 1e-12, s
        assert res_e[s] == stat[s, 1]
        np.testing.assert_array_equal(res_f[rows], forces[rows])
        V = abs(np.linalg.det(cell0[s] @ F[s].T))
        assert rel(res_s[s], bsum[s, 1:] / V * 160.21766208) < 1e-12, s
        assert rel(r0_[rows], o.r0) < 1e-12, s
        assert dt_[s] == pytest.approx(o.dt, rel=1e-15) and a_[s] == pytest.approx(o.a, rel=1e-15), s
        assert ns_[s] == o.nsteps, s
        if flag:
            np.testing.assert_array_equal(v_[rows], v[rows])
            continue
        vref = o.v[:natoms[s]]
        assert rel(v_[rows], vref) < 1e-12, s
        if relax_cell:
            assert rel(vc_[s], o.v[natoms[s]:]) < 1e-12, s
            assert rel(X_[s], o.X) < 1e-12, s
            assert rel(F_[s], expm(o.X / natoms[s])) < 1e-12, s
        assert rel(stat[s, 3:], (o.cell0 @ o.F().T).ravel()) < 1e-12, s


def test_error_after_compaction_names_the_input_index():
    """a structure that loses every edge at step 1, after the first structure left the batch at step 0 (so its batch
    index is 1): the message names its input index, 2, and the step"""
    fam = Family("chgnet")
    rc = fam.model.cutoff
    crystal = si_diamond(2, sigma=0.0)  # forces vanish by symmetry: converges at step 0
    # a repulsive pair just inside the cutoff in a large non-periodic box: one large step moves it out of range
    pair = None
    for r in np.linspace(rc - 0.6, rc - 0.05, 12):
        cand = SimpleAtoms(["Si", "Si"], np.array([[10.0, 10.0, 10.0], [10.0 + r, 10.0, 10.0]]), np.eye(3) * 30.0,
                           pbc=(False, False, False))
        fam.set_structures([cand])
        _, f, _ = fam.eng.compute_batch()
        if f[1, 0] > 1e-3:
            pair = cand
            break
    assert pair is not None, "no repulsive separation near the cutoff"
    moving = mixed(si_diamond(2, sigma=0.15, seed=1))
    with pytest.raises(_lib.B2MError, match="relaxation step 1: structure 2 has no edges") as ei:
        device(fam, [crystal, moving, pair], fmax=5e-4, steps=3, relax_cell=False, dt=100.0, dtmax=100.0, maxstep=2.0)
    assert ei.value.code == B2M_ERR_INVALID
    assert device(fam, [crystal], fmax=0.0, steps=1, relax_cell=False)["steps"][0] == 1  # the handle stays usable


def test_more_c_refusals():
    fam = Family("chgnet")
    a = si_diamond(2, sigma=0.1)
    n, cart, lat, sp, pbc = inputs(fam, [a])
    with pytest.raises(_lib.B2MError, match="fmax must be >= 0"):
        fam.eng.relax_batch(n, cart, lat, sp, pbc, fmax=-1.0)
    with pytest.raises(_lib.B2MError, match="structure 1: no atoms") as ei:
        fam.eng.relax_batch([64, 0], cart, np.array([lat[0], lat[0]]), sp, np.array([pbc[0], pbc[0]]))
    assert ei.value.code == B2M_ERR_INVALID
    # null result pointers through the C-ABI itself
    prm = _lib.RelaxParams(fmax=0.1, steps=1, relax_cell=0, stress_weight=1 / 160.21766208,
                           **{k: float(v) for k, v in FIRE_DEFAULTS.items()})
    n64 = np.array([64], np.int64)
    c_, l_ = np.ascontiguousarray(cart), np.ascontiguousarray(lat.reshape(9))
    sp_, pb_ = np.ascontiguousarray(sp, np.int32), np.ascontiguousarray(pbc.reshape(3), np.int32)
    e = np.zeros(1)
    rc = fam.eng.lib.b2m_relax_batch(fam.eng.h, 1, n64.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                     c_.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                     l_.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                     sp_.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                     pb_.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), 1e-8, ctypes.byref(prm),
                                     e.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None, None, None, None, None)
    assert rc == B2M_ERR_INVALID and b"null result argument" in fam.eng.lib.b2m_last_error(fam.eng.h)
    # weights not finalized
    from tests._util import make_model

    model = make_model(seed=2)
    sd = model.state_dict()
    raw = _lib.Engine(n_elem=sd["atom_embedding.weight"].shape[0], dim=64, max_n=9, max_f=4, n_blocks=model.n_blocks,
                      cutoff=float(model.cutoff), three_body_cutoff=float(model.three_body_cutoff),
                      cutoff_exponent=int(model.cutoff_exponent), device=0)
    with pytest.raises(_lib.B2MError, match="not finalized") as ei:
        raw.relax_batch(n, cart, lat, sp, pbc)
    assert ei.value.code == B2M_ERR_STATE


def test_engine_records_the_resident_batch():
    """after compaction the resident batch is the structures of the last step: compute_batch describes them"""
    fam = Family("chgnet")
    crystal = si_diamond(2, sigma=0.0)  # converges at step 0
    moving = mixed(si_diamond(2, sigma=0.15, seed=1))
    r = device(fam, [moving, crystal, moving], fmax=5e-4, steps=2, relax_cell=False)
    assert list(r["steps"]) == [2, 0, 2]
    assert list(fam.eng.batch_natoms) == [len(moving), len(moving)] and fam.eng.natoms == 2 * len(moving)
    e, f, _ = fam.eng.compute_batch()
    assert e.shape == (2,) and f.shape == (2 * len(moving), 3)
    np.testing.assert_allclose(e, r["energies"][[0, 2]], rtol=1e-8)
