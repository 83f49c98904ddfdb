"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

CPU restatement (torch, float64) of two radial options of mace's `ScaleShiftMACE`, for either hidden shape
(oracle/mace_ref.py: C x 0e; tests/mace_eq_ref.py: C x 0e + C x 1o), with mace's state_dict names: the ZBL pair
repulsion (`pair_repulsion_fn`, mace's `ZBLBasis`) and the Agnesi distance transform of the radial embedding
(`radial_embedding.distance_transform`, mace's `AgnesiTransform`).  Every convention of those two modules holds here
unchanged; with both options off the models below compute exactly what they compute.  mace is not available here, so
what follows is recalled, not pinned against a mace checkout.

Edge e: sender u = src, receiver v = dst, vector v_e = r_v - r_u (+ shift), d = |v_e|, Z the atomic number of an endpoint
(`atomic_numbers[species]`).

  * Agnesi (keys q, p, a, covalent_radii; the radii indexed by Z, ase's 119-entry table in mace's checkpoints):
    r0 = (rho[Z_u] + rho[Z_v]) / 2, s = d / r0, x = 1 + a s^q / (1 + s^(q - p)).  The radial features become
    ef_n = b_n(x) f_cut(d): the Bessel basis (same weights and prefactor) takes x, the polynomial cutoff keeps d and r_max.
  * ZBL (keys c [4], a_exp, a_prefactor, p, covalent_radii):
    a_uv = a_prefactor 0.529 / (Z_u^a_exp + Z_v^a_exp), t = d / a_uv,
    phi = c0 e^(-3.2 t) + c1 e^(-0.9423 t) + c2 e^(-0.4029 t) + c3 e^(-0.2016 t),
    V_e = 1/2 14.3996 Z_u Z_v / d phi env_p(d / (rho'[Z_u] + rho'[Z_v])), env_p mace's PolynomialCutoff envelope with
    exponent p (zero at and beyond 1).  e_pair(i) = sum over the edges e with dst(e) = i of V_e (each pair is two directed
    edges, so this is 1/2 sum_j V_ij).  A ZBL cutoff larger than r_max stays as it is: edges only exist within r_max.
  * energy of atom i: E0[z_i] + scale (e_pair(i) + sum_t e_t(i)) + shift -- the pair energy is inside scale, and first in
    the sum, as mace lists it first among the node energies.

The covalent-radius table below (Cordero et al. 2008, the values ase ships, recalled; 0.2 where ase has no value) only
has to be plausible: the engine reads whatever table the state_dict holds.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from oracle import mace_ref as _s
from tests import mace_eq_ref as _eq

COVALENT_RADII = np.array([
    0.20, 0.31, 0.28, 1.28, 0.96, 0.84, 0.76, 0.71, 0.66, 0.57, 0.58,            # X, H .. Ne
    1.66, 1.41, 1.21, 1.11, 1.07, 1.05, 1.02, 1.06,                              # Na .. Ar
    2.03, 1.76, 1.70, 1.60, 1.53, 1.39, 1.39, 1.32, 1.26, 1.24, 1.32, 1.22,      # K .. Zn
    1.22, 1.20, 1.19, 1.20, 1.20, 1.16,                                          # Ga .. Kr
    2.20, 1.95, 1.90, 1.75, 1.64, 1.54, 1.47, 1.46, 1.42, 1.39, 1.45, 1.44,      # Rb .. Cd
    1.42, 1.39, 1.39, 1.38, 1.39, 1.40,                                          # In .. Xe
    2.44, 2.15, 2.07, 2.04, 2.03, 2.01, 1.99, 1.98, 1.98, 1.96, 1.94, 1.92,      # Cs .. Dy
    1.92, 1.89, 1.90, 1.87, 1.87, 1.75, 1.70, 1.62, 1.51, 1.44, 1.41, 1.36,      # Ho .. Pt
    1.36, 1.32, 1.45, 1.46, 1.48, 1.40, 1.50, 1.50,                              # Au .. Rn
    2.60, 2.21, 2.15, 2.06, 2.00, 1.96, 1.90, 1.87, 1.80, 1.69] + [0.20] * 22)   # Fr .. Cm, Bk .. Og
assert COVALENT_RADII.shape == (119,)

ZBL_C = (0.1818, 0.5099, 0.2802, 0.02817)


class AgnesiTransform(nn.Module):
    def __init__(self, q=0.9183, p=4.5791, a=1.0805):
        super().__init__()
        self.register_buffer("q", torch.tensor(q, dtype=torch.float64))
        self.register_buffer("p", torch.tensor(p, dtype=torch.float64))
        self.register_buffer("a", torch.tensor(a, dtype=torch.float64))
        self.register_buffer("covalent_radii", torch.tensor(COVALENT_RADII, dtype=torch.float64))

    def forward(self, d, Zu, Zv):  # d [E, 1], Z [E] (int64) -> x [E, 1]
        r0 = 0.5 * (self.covalent_radii[Zu] + self.covalent_radii[Zv])[:, None]
        s = d / r0
        return 1.0 + self.a * s ** self.q / (1.0 + s ** (self.q - self.p))


class ZBLBasis(nn.Module):
    def __init__(self, p=6):
        super().__init__()
        self.register_buffer("c", torch.tensor(ZBL_C, dtype=torch.float64))
        self.register_buffer("a_exp", torch.tensor(0.300, dtype=torch.float64))
        self.register_buffer("a_prefactor", torch.tensor(0.4543, dtype=torch.float64))
        self.register_buffer("p", torch.tensor(float(p), dtype=torch.float64))
        self.register_buffer("covalent_radii", torch.tensor(COVALENT_RADII, dtype=torch.float64))

    def edge_energies(self, d, Zu, Zv):  # d [E], Z [E] (int64) -> V_e [E]
        zu, zv = Zu.to(d.dtype), Zv.to(d.dtype)
        a = self.a_prefactor * 0.529 / (zu ** self.a_exp + zv ** self.a_exp)
        t = d / a
        c = self.c
        phi = c[0] * torch.exp(-3.2 * t) + c[1] * torch.exp(-0.9423 * t) + c[2] * torch.exp(-0.4029 * t) + \
            c[3] * torch.exp(-0.2016 * t)
        rc = self.covalent_radii[Zu] + self.covalent_radii[Zv]
        return 0.5 * 14.3996 * zu * zv / d * phi * _s.polynomial_cutoff(d, rc, self.p)

    def forward(self, d, Zu, Zv, dst, n):  # e_pair [n]
        return torch.zeros(n, dtype=d.dtype).index_add(0, dst, self.edge_energies(d, Zu, Zv))


class RadialEmbeddingBlock(_s.RadialEmbeddingBlock):
    """Bessel x polynomial cutoff; with a transform the Bessel basis takes x(d, Z_u, Z_v) and the cutoff keeps d"""

    def __init__(self, r_max, num_bessel, p, distance_transform=None):
        super().__init__(r_max, num_bessel, p)
        self.distance_transform = distance_transform

    def forward(self, d, Zu=None, Zv=None):
        if self.distance_transform is None:
            return super().forward(d)
        return self.bessel_fn(self.distance_transform(d, Zu, Zv)) * self.cutoff_fn(d)


class _CoreRepulsion:
    """node_energies of both ScaleShiftMACE restatements with the pair term and the transform"""

    def _add_options(self, pair_repulsion, distance_transform):
        old = self.radial_embedding
        r_max, nb, p = float(old.bessel_fn.r_max), old.bessel_fn.bessel_weights.numel(), float(old.cutoff_fn.p)
        self.radial_embedding = RadialEmbeddingBlock(r_max, nb, p, distance_transform)
        self.radial_embedding.load_state_dict(old.state_dict(), strict=False)
        self.pair_repulsion = bool(pair_repulsion)
        if pair_repulsion:
            self.pair_repulsion_fn = ZBLBasis()

    def node_energies(self, vec, src, dst, z, taps=None):
        """(eps_i [n], interaction part e_i [n]) as the model without the options computes them, plus the pair term"""
        d = torch.linalg.norm(vec, dim=1, keepdim=True)
        Zn = self.atomic_numbers[z]
        Y = _s.sh_basis(vec, self.max_ell)
        if self.radial_embedding.distance_transform is None:
            ef = self.radial_embedding(d)
        else:
            ef = self.radial_embedding(d, Zn[src], Zn[dst])
        if taps is not None:
            taps["eb"] = ef.detach()
        h = self.node_embedding(z)
        e = torch.zeros(z.shape[0], dtype=vec.dtype)
        if self.pair_repulsion:
            pair = self.pair_repulsion_fn(d[:, 0], Zn[src], Zn[dst], dst, z.shape[0])
            e = e + pair
            if taps is not None:
                taps["e_pair"] = pair.detach()
        for t, (inter, prod, ro) in enumerate(zip(self.interactions, self.products, self.readouts)):
            A, sc = inter(h, z, Y, ef, src, dst)
            h = prod(A, sc, z)
            e = e + ro(h)
            if taps is not None:
                taps[f"A{t}"], taps[f"h{t + 1}"] = A.detach(), h.detach()
        inter_e = self.scale_shift.scale * e + self.scale_shift.shift
        return self.atomic_energies_fn.atomic_energies[z] + inter_e, inter_e


class ScaleShiftMACE(_CoreRepulsion, _s.ScaleShiftMACE):
    """oracle/mace_ref.py ScaleShiftMACE (C x 0e) with mace's pair_repulsion and distance_transform options"""

    def __init__(self, atomic_numbers, pair_repulsion=False, distance_transform=None, **kw):
        super().__init__(atomic_numbers, **kw)
        self._add_options(pair_repulsion, distance_transform)


class ScaleShiftMACEEq(_CoreRepulsion, _eq.ScaleShiftMACE):
    """tests/mace_eq_ref.py ScaleShiftMACE (C x 0e + C x 1o) with the same options"""

    def __init__(self, atomic_numbers, pair_repulsion=False, distance_transform=None, **kw):
        super().__init__(atomic_numbers, **kw)
        self._add_options(pair_repulsion, distance_transform)


def _make(cls, seed, atomic_numbers, pair_repulsion, distance_transform, kw):
    torch.manual_seed(seed)  # the options carry no random weights: the rest is the model the base factory builds
    kw.setdefault("atomic_energies", np.linspace(-3.0, -1.0, len(atomic_numbers)))
    kw.setdefault("scale", 1.3)
    kw.setdefault("shift", -0.2)
    if distance_transform == "agnesi":
        distance_transform = AgnesiTransform()
    return cls(list(atomic_numbers), pair_repulsion=pair_repulsion, distance_transform=distance_transform, **kw)


def make_mace(seed=0, atomic_numbers=(14, 6, 8), pair_repulsion=False, distance_transform=None, **kw):
    """oracle/mace_ref.py make_mace with mace's opt-in radial options (distance_transform: None, "agnesi" or a module)"""
    return _make(ScaleShiftMACE, seed, atomic_numbers, pair_repulsion, distance_transform, kw)


def make_mace_eq(seed=0, atomic_numbers=(14, 6, 8), pair_repulsion=False, distance_transform=None, **kw):
    """tests/mace_eq_ref.py make_mace_eq with the same options"""
    return _make(ScaleShiftMACEEq, seed, atomic_numbers, pair_repulsion, distance_transform, kw)


potential_ref = _s.potential_ref
atomic_virials_ref = _s.atomic_virials_ref
