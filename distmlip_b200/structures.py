"""Deterministic synthetic structures used by tests and bench.py (SURVEY.md §8d).

No external data: everything here is generated from a seed.  ASE / pymatgen are
not available in this image, so `SimpleAtoms` duck-types the handful of
`ase.Atoms` methods the reference's hot path touches
(reference: DistMLIP/implementations/matgl/pes.py:69-73, models/chgnet.py:44-46,66-69).
"""
from __future__ import annotations

import numpy as np

SI_A = 5.431  # Angstrom, diamond-cubic Si conventional cell

SYMBOLS = (
    "X H He Li Be B C N O F Ne Na Mg Al Si P S Cl Ar K Ca Sc Ti V Cr Mn Fe Co Ni Cu Zn Ga Ge As Se Br Kr Rb Sr Y Zr "
    "Nb Mo Tc Ru Rh Pd Ag Cd In Sn Sb Te I Xe Cs Ba La Ce Pr Nd Pm Sm Eu Gd Tb Dy Ho Er Tm Yb Lu Hf Ta W Re Os Ir Pt "
    "Au Hg Tl Pb Bi Po At Rn Fr Ra Ac Th Pa U Np Pu Am Cm Bk Cf Es Fm Md No Lr Rf Db Sg Bh Hs Mt Ds Rg Cn Nh Fl Mc Lv "
    "Ts Og").split()
Z_OF = {s: z for z, s in enumerate(SYMBOLS)}

_DIAMOND_BASIS = np.array(
    [
        [0.00, 0.00, 0.00],
        [0.00, 0.50, 0.50],
        [0.50, 0.00, 0.50],
        [0.50, 0.50, 0.00],
        [0.25, 0.25, 0.25],
        [0.25, 0.75, 0.75],
        [0.75, 0.25, 0.75],
        [0.75, 0.75, 0.25],
    ]
)


class SimpleAtoms:
    """Minimal stand-in for ase.Atoms (same method names / return conventions)."""

    def __init__(self, symbols, positions, cell, pbc=(True, True, True)):
        self._symbols = list(symbols)
        self._positions = np.ascontiguousarray(positions, dtype=np.float64)
        self._cell = np.ascontiguousarray(cell, dtype=np.float64).reshape(3, 3)
        self._pbc = np.array(pbc, dtype=bool)

    def __len__(self):
        return len(self._symbols)

    def get_cell(self):
        return self._cell.copy()

    def get_positions(self, wrap=False):
        if not wrap:
            return self._positions.copy()
        return self.get_scaled_positions(wrap=True) @ self._cell

    def set_positions(self, pos):
        self._positions = np.ascontiguousarray(pos, dtype=np.float64)

    def set_cell(self, cell, scale_atoms=False):
        cell = np.ascontiguousarray(cell, dtype=np.float64).reshape(3, 3)
        if scale_atoms:
            self._positions = np.linalg.solve(self._cell.T, self._positions.T).T @ cell
        self._cell = cell

    def get_scaled_positions(self, wrap=True):
        frac = np.linalg.solve(self._cell.T, self._positions.T).T
        if wrap:
            for i in range(3):
                if self._pbc[i]:
                    frac[:, i] %= 1.0
                    frac[:, i] %= 1.0
        return frac

    def get_pbc(self):
        return self._pbc.copy()

    def get_chemical_symbols(self):
        return list(self._symbols)

    @property
    def positions(self):  # ase.Atoms.positions: the internal array, no copy
        return self._positions

    @property
    def numbers(self):  # ase.Atoms.numbers
        if getattr(self, "_numbers", None) is None:
            self._numbers = np.array([Z_OF[s] for s in self._symbols], dtype=np.int64)
        return self._numbers

    def get_atomic_numbers(self):
        if getattr(self, "_numbers", None) is None:
            self._numbers = np.array([Z_OF[s] for s in self._symbols], dtype=np.int64)
        return self._numbers.copy()

    def get_volume(self):
        return float(abs(np.linalg.det(self._cell)))


def si_diamond(n, sigma=0.15, seed=0, nz=None, symbol="Si"):
    """Perturbed diamond-cubic Si, n x n x (nz or n) conventional cells (8 atoms each).

    frac = ((cell + basis)/n + N(0, sigma^2)/(a n)) mod 1, numpy default_rng(seed)
    (SURVEY.md §8d).  Returns SimpleAtoms.
    """
    nz = n if nz is None else nz
    rng = np.random.default_rng(seed)
    gx, gy, gz = np.meshgrid(np.arange(n), np.arange(n), np.arange(nz), indexing="ij")
    cells = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], axis=1).astype(np.float64)
    dims = np.array([n, n, nz], dtype=np.float64)
    frac = (cells[:, None, :] + _DIAMOND_BASIS[None, :, :]).reshape(-1, 3) / dims
    lattice = np.diag(dims * SI_A)
    if sigma > 0:
        frac = frac + rng.normal(0.0, sigma, size=frac.shape) / (SI_A * dims)
    frac %= 1.0
    frac %= 1.0
    pos = frac @ lattice
    return SimpleAtoms([symbol] * len(pos), pos, lattice)


def rough_cell(natoms, density=0.05, min_dist=2.2, seed=0, symbol="Si", aspect=(1, 1, 1)):
    """Random sequential addition structure (degree-imbalance stress case, SURVEY §8d)."""
    rng = np.random.default_rng(seed)
    vol = natoms / density
    asp = np.array(aspect, dtype=np.float64)
    s = (vol / asp.prod()) ** (1.0 / 3.0)
    L = asp * s
    lattice = np.diag(L)
    ncell = np.maximum(1, np.floor(L / min_dist).astype(int))
    grid = {}
    pts = []
    tries = 0
    while len(pts) < natoms and tries < natoms * 200:
        tries += 1
        p = rng.random(3) * L
        c = tuple((p / L * ncell).astype(int) % ncell)
        ok = True
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    cc = ((c[0] + dx) % ncell[0], (c[1] + dy) % ncell[1], (c[2] + dz) % ncell[2])
                    for q in grid.get(cc, ()):
                        d = p - q
                        d -= np.round(d / L) * L
                        if d @ d < min_dist * min_dist:
                            ok = False
                            break
                    if not ok:
                        break
                if not ok:
                    break
            if not ok:
                break
        if ok:
            grid.setdefault(c, []).append(p)
            pts.append(p)
    pos = np.array(pts)
    return SimpleAtoms([symbol] * len(pos), pos, lattice)
