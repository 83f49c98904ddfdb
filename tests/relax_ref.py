"""float64 restatement of the batched relaxation (DESIGN.md §13): ASE's FIRE with, optionally, its FrechetCellFilter
(exp_cell_factor = natoms, scalar_pressure), one independent optimizer per structure, driven by a force callback.

The cell force uses scipy's `expm_frechet` nine times, as ASE does, so that it is independent of the engine's 6x6
adjoint form.  A structure's generalised coordinates are its reference positions r0 [n, 3] and, with the filter, the
three rows X = n logm(F) (kept as state, X = 0 at the start); the geometry is r0 F^T, cell0 F^T with F = expm(X / n).
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import expm, expm_frechet

FIRE_DEFAULTS = dict(dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)


def cell_force(X, W, V, n, k=1.0, p=0.0):
    """generalised force on the cell rows: W [3, 3] the strain derivative of the energy (eV), V the current volume,
    k its weight, p the scalar pressure (eV/A^3) -- ase.filters.FrechetCellFilter.get_forces"""
    F = expm(X / n)
    virial = -(k * 0.5 * (W + W.T) + p * V * np.eye(3))
    virial = np.linalg.solve(F, virial.T).T
    out = np.zeros((3, 3))
    for mu in range(3):
        for nu in range(3):
            d = np.zeros((3, 3))
            d[mu, nu] = 1.0
            out[mu, nu] = np.sum(expm_frechet(X / n, d, compute_expm=False) * virial)
    return out / n


class Fire:
    """one structure's optimizer (ase.optimize.FIRE + FrechetCellFilter), state in f64"""

    def __init__(self, pos, cell, relax_cell, k=1.0, p=0.0, **fire):
        c = dict(FIRE_DEFAULTS, **fire)
        self.c = c
        self.r0 = np.array(pos, dtype=np.float64).reshape(-1, 3)
        self.cell0 = np.array(cell, dtype=np.float64).reshape(3, 3)
        self.n = len(self.r0)
        self.relax_cell, self.k, self.p = relax_cell, k, p
        self.X = np.zeros((3, 3))
        self.v = None
        self.dt, self.a, self.nsteps = c["dt"], c["a"], 0
        self.margins = []  # |P| / (|f| |v|) of every FIRE branch taken

    def F(self):
        return expm(self.X / self.n) if self.relax_cell else np.eye(3)

    def geometry(self):
        F = self.F()
        return self.r0 @ F.T, self.cell0 @ F.T

    def forces(self, f, W):
        """generalised forces [n (+ 3), 3] from the engine's forces f [n, 3] and strain derivative W [3, 3]"""
        F = self.F()
        g = np.asarray(f, dtype=np.float64) @ F
        if not self.relax_cell:
            return g
        V = abs(np.linalg.det(self.cell0 @ F.T))
        return np.vstack([g, cell_force(self.X, W, V, self.n, self.k, self.p)])

    def step(self, f):
        c = self.c
        if self.v is None:
            self.v = np.zeros_like(f)
        else:
            vf = np.vdot(f, self.v)
            self.margins.append(abs(vf) / (np.sqrt(np.vdot(f, f)) * np.sqrt(np.vdot(self.v, self.v)) + 1e-300))
            if vf > 0.0:
                self.v = (1.0 - self.a) * self.v + self.a * f / np.sqrt(np.vdot(f, f)) * np.sqrt(np.vdot(self.v, self.v))
                if self.nsteps > c["Nmin"]:
                    self.dt = min(self.dt * c["finc"], c["dtmax"])
                    self.a *= c["fa"]
                self.nsteps += 1
            else:
                self.v[:] *= 0.0
                self.a = c["astart"]
                self.dt *= c["fdec"]
                self.nsteps = 0
        self.v += self.dt * f
        dr = self.dt * self.v
        normdr = np.sqrt(np.vdot(dr, dr))
        if normdr > c["maxstep"]:
            dr = c["maxstep"] * dr / normdr
        self.r0 = self.r0 + dr[:self.n]
        if self.relax_cell:
            self.X = self.X + dr[self.n:]


def relax(structures, evaluate, fmax, steps, relax_cell, p=0.0, k=1.0, **fire):
    """ase Optimizer.run per structure: evaluate, stop when max row |f| < fmax or after `steps` steps, else step.
    structures: list of (positions [n, 3], cell [3, 3]); evaluate(ids, geometries) -> list of (energy, forces [n, 3],
    W [3, 3]) for the structures ids at geometries [(positions, cell)].  Returns one dict per structure: positions,
    cell, energy, forces, W (of the last evaluation), steps, converged, and per evaluation energies, max row forces
    (fmaxes) and geometries (positions, cell), and the margins of the FIRE branches."""
    opt = [Fire(x, c, relax_cell, k=k, p=p, **fire) for x, c in structures]
    out = [dict(energies=[], geometries=[], fmaxes=[], steps=None, converged=False) for _ in structures]
    active = list(range(len(structures)))
    for it in range(steps + 1):
        if not active:
            break
        geos = [opt[s].geometry() for s in active]
        res = evaluate(active, geos)
        still = []
        for s, geo, (E, f, W) in zip(active, geos, res):
            o = out[s]
            o.update(positions=geo[0], cell=geo[1], energy=float(E), forces=np.asarray(f), W=np.asarray(W))
            o["energies"].append(float(E))
            o["geometries"].append(geo)
            g = opt[s].forces(f, W)
            o["fmaxes"].append(float(np.sqrt((g ** 2).sum(axis=1).max())))
            if (g ** 2).sum(axis=1).max() < fmax ** 2:
                o.update(steps=it, converged=True)
                continue
            if it == steps:
                o.update(steps=it, converged=False)
                continue
            opt[s].step(g)
            still.append(s)
        active = still
    for s, o in enumerate(out):
        o["margins"] = opt[s].margins
    return out


# ---------------------------------------------------------------- Lennard-Jones in numpy (tests' analytic potential)
def lj(pos, cell, sigma=2.0, eps=0.05, rc=5.0):
    """energy, forces [n, 3] and strain derivative W [3, 3] of a truncated, shifted Lennard-Jones solid (periodic)"""
    pos = np.asarray(pos, dtype=np.float64)
    cell = np.asarray(cell, dtype=np.float64)
    inv = np.linalg.inv(cell)
    heights = 1.0 / np.linalg.norm(inv, axis=0)
    m = np.ceil(rc / heights).astype(int) + 1
    shifts = np.array([[i, j, k] for i in range(-m[0], m[0] + 1) for j in range(-m[1], m[1] + 1)
                       for k in range(-m[2], m[2] + 1)], dtype=np.float64) @ cell
    d = pos[None, :, None, :] - pos[:, None, None, :] + shifts[None, None, :, :]  # [i, j, image, 3]: r_j + T - r_i
    r = np.linalg.norm(d, axis=-1)
    mask = (r < rc) & (r > 1e-8)
    rs = np.where(mask, r, 1.0)
    sr6 = (sigma / rs) ** 6
    src6 = (sigma / rc) ** 6
    phi = np.where(mask, 4 * eps * (sr6 * sr6 - sr6) - 4 * eps * (src6 * src6 - src6), 0.0)
    dphi = np.where(mask, 4 * eps * (-12 * sr6 * sr6 + 6 * sr6) / rs, 0.0)  # dphi/dr
    E = 0.5 * phi.sum()
    fij = (dphi / rs)[..., None] * d  # dphi/dr * unit(r_j - r_i): pulls i toward j when dphi > 0
    forces = fij.sum(axis=(1, 2))
    W = 0.5 * np.einsum("ijt,ijta,ijtb->ab", dphi / rs, d, d)
    return E, forces, W


def fcc(a, reps=2):
    base = np.array([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]])
    grid = np.array([[i, j, k] for i in range(reps) for j in range(reps) for k in range(reps)])
    frac = (base[None, :, :] + grid[:, None, :]).reshape(-1, 3) / reps
    cell = np.eye(3) * a * reps
    return frac @ cell, cell
