"""CPU checks of the ZBL pair repulsion and the Agnesi distance transform in the MACE oracle (tests/mace_zbl_ref.py), of
the wrapper's configuration checks for them, and of the margin between the GPU tolerances and plausible bugs."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from distmlip_b200.structures import Z_OF, SimpleAtoms, rough_cell, si_diamond
from oracle.mace_ref import make_mace as make_plain
from tests.mace_eq_ref import make_mace_eq as make_plain_eq
from tests.mace_zbl_ref import (COVALENT_RADII, ZBL_C, atomic_virials_ref, make_mace, make_mace_eq, potential_ref)

SYMS = ("H", "O", "Si", "Fe")  # Z_u Z_v from 1 to 676
ZS = tuple(Z_OF[s] for s in SYMS)
OPTIONS = {"zbl": dict(pair_repulsion=True), "agnesi": dict(distance_transform="agnesi"),
           "both": dict(pair_repulsion=True, distance_transform="agnesi")}
# the thresholds of tests/test_gpu_mace*.py: energy per atom, forces, stress (GPa), per-atom energies
TOL = {"e": 1e-4, "f": 1e-3, "s": 1e-3, "eps": 1e-4}


def mixed(atoms, seed=0, syms=SYMS):
    rng = np.random.default_rng(seed)
    sy = [syms[k] for k in rng.integers(0, len(syms), len(atoms))]
    return SimpleAtoms(sy, atoms.get_positions(), np.array(atoms.get_cell()), pbc=atoms.get_pbc())


def model(opt="both", eq=False, **kw):
    """the GPU tests' models: C = 32, r_max 6, scale 8, species H, O, Si, Fe"""
    kw.setdefault("C", 32)
    kw.setdefault("r_max", 6.0)
    kw.setdefault("scale", 8.0)
    kw.setdefault("atomic_numbers", ZS)
    kw.update(OPTIONS[opt] if opt else {})
    return (make_mace_eq if eq else make_mace)(**kw)


# the GPU tests' structures
def diamond64():
    return mixed(si_diamond(2, seed=1))


def close_contact():
    return mixed(rough_cell(100, min_dist=0.7, seed=3), seed=4)


def dimer(d, a="Si", b="Fe"):
    return SimpleAtoms([a, b], np.array([[10.0, 10.0, 10.0], [10.0 + d, 10.0, 10.0]]), np.eye(3) * 30.0,
                       pbc=(False, False, False))


def cluster():
    a = si_diamond(2, seed=4)
    return mixed(SimpleAtoms(["Si"] * len(a), a.get_positions(), np.eye(3) * 40.0, pbc=(False, False, False)), seed=3)


# ---------------------------------------------------------------------------------------------- closed forms
def zbl_pair_numpy(d, z1, z2, p=6):
    """the ZBL energy of a pair (both directed edges) from the formula, numpy only"""
    a = 0.4543 * 0.529 / (z1 ** 0.3 + z2 ** 0.3)
    t = d / a
    phi = sum(c * np.exp(-b * t) for c, b in zip(ZBL_C, (3.2, 0.9423, 0.4029, 0.2016)))
    x = d / (COVALENT_RADII[z1] + COVALENT_RADII[z2])
    env = (1 - 0.5 * (p + 1) * (p + 2) * x ** p + p * (p + 2) * x ** (p + 1) - 0.5 * p * (p + 1) * x ** (p + 2)) * (x < 1)
    return 14.3996 * z1 * z2 / d * phi * env


@pytest.mark.parametrize("pair", [("Si", "Si"), ("H", "Fe"), ("O", "Si"), ("Fe", "Fe")])
def test_zbl_dimer_closed_form(pair):
    m, m0 = model("zbl"), model(None)
    z1, z2 = Z_OF[pair[0]], Z_OF[pair[1]]
    rc = COVALENT_RADII[z1] + COVALENT_RADII[z2]
    for d in np.concatenate([np.linspace(0.4, 3.0, 8), [rc - 1e-3, rc + 1e-3, 4.0]]):
        a = dimer(d, *pair)
        dE = (potential_ref(m, a, calc_forces=False)[0] - potential_ref(m0, a, calc_forces=False)[0]).item() / 8.0
        want = zbl_pair_numpy(d, z1, z2)
        assert abs(dE - want) < 1e-10 * max(1.0, abs(want)), (d, dE, want)
        if d > rc:
            assert dE == 0.0
    assert zbl_pair_numpy(0.5, z1, z2) > 1.0


def test_agnesi_radial_features_closed_form():
    m = model("agnesi", num_bessel=8)
    atoms = mixed(si_diamond(1, seed=2), seed=1)
    taps = {}
    potential_ref(m, atoms, calc_forces=False, taps=taps)
    from oracle.graph_ref import neighbor_list

    i1, i2, off, _, _ = neighbor_list(atoms.get_positions(), np.array(atoms.get_cell()), atoms.get_pbc().astype(np.int64),
                                      6.0, 0.0)
    pos = atoms.get_positions()
    d = np.linalg.norm(pos[i2] + off @ np.array(atoms.get_cell()) - pos[i1], axis=1)
    z = atoms.get_atomic_numbers()
    r0 = 0.5 * (COVALENT_RADII[z[i1]] + COVALENT_RADII[z[i2]])
    s = d / r0
    q, p, a = 0.9183, 4.5791, 1.0805
    x = 1 + a * s ** q / (1 + s ** (q - p))
    w = np.pi / 6.0 * np.arange(1, 9)
    u = d / 6.0
    f = (1 - 21 * u ** 5 + 35 * u ** 6 - 15 * u ** 7) * (u < 1)
    want = np.sqrt(2 / 6.0) * np.sin(w[None] * x[:, None]) / x[:, None] * f[:, None]
    assert np.abs(taps["eb"].numpy() - want).max() < 1e-12
    assert np.abs(x - d).max() > 0.1  # the transform moves the basis


# ---------------------------------------------------------------------------------------------- derivatives
def small(seed=0):
    a = si_diamond(1, seed=seed, sigma=0.3)  # 8 atoms, 5.43 A cell, pushed together
    return mixed(SimpleAtoms(a.get_chemical_symbols(), a.get_positions() * 0.8, np.array(a.get_cell()) * 0.8), seed)


@pytest.mark.parametrize("eq", [False, True], ids=["0e", "0e+1o"])
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_forces_stress_finite_differences(opt, eq):
    m = model(opt, eq=eq, r_max=4.0, scale=1.3, seed=3)
    a = small(seed=5)
    E, F, S, eps = potential_ref(m, a)
    taps = {}
    potential_ref(m, a, calc_forces=False, taps=taps)
    if "pair_repulsion" in OPTIONS[opt]:
        assert taps["e_pair"].abs().max() > 1e-2  # the pair term is active in this cell
    h = 1e-5
    pos, cell = a.get_positions(), np.array(a.get_cell())
    en = lambda p, c: potential_ref(m, SimpleAtoms(a.get_chemical_symbols(), p, c), calc_forces=False,  # noqa: E731
                                    calc_stresses=False)[0].item()
    for i, k in ((0, 0), (5, 2)):
        dp = np.zeros_like(pos)
        dp[i, k] = h
        fd = -(en(pos + dp, cell) - en(pos - dp, cell)) / (2 * h)
        assert abs(fd - F[i, k].item()) < 1e-6 * max(1.0, abs(fd)), (fd, F[i, k].item())
    eps_m = np.zeros((3, 3))
    eps_m[1, 2] = eps_m[2, 1] = h / 2
    fd = (en(pos @ (np.eye(3) + eps_m), cell @ (np.eye(3) + eps_m)) -
          en(pos @ (np.eye(3) - eps_m), cell @ (np.eye(3) - eps_m))) / (2 * h)
    vol = abs(np.linalg.det(cell))
    assert abs(fd / vol * 160.21766208 - S[1, 2].item()) < 1e-5 * max(1.0, abs(S[1, 2].item()))
    # sum rules: per-atom energies and per-atom virials
    assert abs(eps.sum().item() - E.item()) < 1e-10 * max(1.0, abs(E.item()))
    w = atomic_virials_ref(m, a).numpy()
    np.testing.assert_allclose(w.sum(axis=0), S.numpy() * vol / 160.21766208, atol=1e-9 * max(1.0, np.abs(w).max()))


@pytest.mark.parametrize("eq", [False, True], ids=["0e", "0e+1o"])
def test_default_off_is_bit_identical(eq):
    a = small(seed=6)
    kw = dict(C=32, r_max=4.0, seed=7, atomic_numbers=ZS)
    base = (make_plain_eq if eq else make_plain)(**kw)
    new = (make_mace_eq if eq else make_mace)(**kw)
    E0, F0, S0, e0 = potential_ref(base, a)
    E1, F1, S1, e1 = potential_ref(new, a)
    assert torch.equal(E0, E1) and torch.equal(F0, F1) and torch.equal(S0, S1) and torch.equal(e0, e1)
    assert list(base.state_dict()) == list(new.state_dict())


# ---------------------------------------------------------------------------------------------- wrapper
def _describe(m):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    return ScaleShiftMACE_Dist.from_existing(m)._describe()


@pytest.mark.parametrize("eq", [False, True], ids=["0e", "0e+1o"])
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_wrapper_accepts(opt, eq):
    desc = _describe(model(opt, eq=eq))
    assert desc.hidden_max_l == int(eq) and desc.n_elem == 4


def _reject(m, match, edit=None):
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    d = ScaleShiftMACE_Dist.from_existing(m)
    if edit is not None:
        edit(d._state_dict)
    with pytest.raises(NotImplementedError, match=match):
        d._describe()


def test_wrapper_refusals_name_the_option():
    m = model("both")
    m.heads = ["a", "b"]
    _reject(m, "multi-head")
    m = model("zbl")
    m.radial_embedding.distance_transform = torch.nn.Identity()  # mace's SoftTransform and others
    _reject(m, "distance_transform Identity")
    m = model("both")
    m.radial_embedding.apply_cutoff = False
    _reject(m, "apply_cutoff")
    m = model(None)
    m.pair_repulsion = True
    _reject(m, "pair_repulsion = True without")
    _reject(model("zbl"), "pair_repulsion_fn.r_max", lambda sd: sd.__setitem__("pair_repulsion_fn.r_max", torch.ones(1)))
    _reject(model("zbl"), "pair_repulsion_fn.a_exp is missing", lambda sd: sd.pop("pair_repulsion_fn.a_exp"))
    _reject(model("zbl"), "4 coefficients", lambda sd: sd.__setitem__("pair_repulsion_fn.c", torch.ones(3)))
    _reject(model("agnesi"), "AgnesiTransform", lambda sd: sd.pop("radial_embedding.distance_transform.q"))
    _reject(model("agnesi"), "AgnesiTransform",
            lambda sd: sd.__setitem__("radial_embedding.distance_transform.b", torch.ones(1)))


# ---------------------------------------------------------------------------------------------- margins
def _mutant(m, kind):
    """a plausible bug, applied to the oracle model in place"""
    if kind == "pair_outside_scale":  # eps = E0 + scale e + shift + e_pair
        orig = m.node_energies

        def ne(vec, src, dst, z, taps=None):
            eps, ie = orig(vec, src, dst, z, taps)
            Zn = m.atomic_numbers[z]
            pair = m.pair_repulsion_fn(torch.linalg.norm(vec, dim=1), Zn[src], Zn[dst], dst, z.shape[0])
            return eps + (1.0 - m.scale_shift.scale) * pair, ie
        m.node_energies = ne
    elif kind == "half_dropped":
        zb = m.pair_repulsion_fn
        orig_e = zb.edge_energies
        zb.edge_energies = lambda d, Zu, Zv: 2.0 * orig_e(d, Zu, Zv)
    elif kind == "cutoff_on_x":
        re = m.radial_embedding
        re.forward = lambda d, Zu=None, Zv=None: (lambda x: re.bessel_fn(x) * re.cutoff_fn(x))(
            re.distance_transform(d, Zu, Zv))
    elif kind == "r0_without_half":  # r0 = rho_u + rho_v
        m.radial_embedding.distance_transform.covalent_radii.mul_(2.0)
    elif kind == "zbl_envelope_on_r_max":  # rho'_u + rho'_v = r_max
        m.pair_repulsion_fn.covalent_radii.fill_(0.5 * float(m.r_max))
    return m


MUTANTS = {"pair_outside_scale": "zbl", "half_dropped": "zbl", "zbl_envelope_on_r_max": "zbl",
           "cutoff_on_x": "agnesi", "r0_without_half": "agnesi"}


def _margin(m, bug, atoms):
    """the largest ratio bug error / GPU tolerance over energy per atom, forces, stress and per-atom energies"""
    E, F, S, eps = potential_ref(m, atoms)
    Eb, Fb, Sb, epsb = potential_ref(bug, atoms)
    n = len(atoms)
    r = [abs(E - Eb).item() / n / TOL["e"], (F - Fb).abs().max().item() / TOL["f"],
         (epsb - eps).abs().max().item() / TOL["eps"]]
    if all(atoms.get_pbc()):
        r.append((S - Sb).abs().max().item() / TOL["s"])
    return max(r)


@pytest.mark.parametrize("kind", list(MUTANTS))
def test_gpu_tolerances_catch_plausible_bugs(kind):
    opt = MUTANTS[kind]
    # the dimer scan of the GPU tests runs the pair term alone (a ZBL-only model)
    for atoms in (diamond64(), close_contact(), cluster()) + ((dimer(1.2), dimer(1.5, "O", "Fe")) if opt == "zbl" else ()):
        m = model(opt, seed=21)
        bug = _mutant(model(opt, seed=21), kind)
        ratio = _margin(m, bug, atoms)
        assert ratio >= 10.0, (kind, len(atoms), ratio)
