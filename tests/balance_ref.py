"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

CPU restatement (numpy, float64 / int64) of the engine's balanced partition policy (graph.cu, DESIGN.md §4.1), which
the reference does not have: the work of every atom from oracle/graph_ref's neighbour and bond lists, the walls at the
work quantiles with the minimum slab width, and GraphOracle with given walls.  engine_inv3 / engine_wrap reproduce the
engine's lattice inverse and wrapped fractional coordinates bit for bit, so that walls placed half-way between two atoms'
coordinates can be compared bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle.graph_ref import EPSILON, GraphOracle, which_partition


class SlabWidthError(ValueError):
    """a balanced partition cannot give every slab the minimum width; `slab` names the first one too thin"""

    def __init__(self, slab, width, need):
        super().__init__(f"slab {slab} is {width:.4f} A wide across the walls < {need:.4f}")
        self.slab, self.width, self.need = slab, width, need


def engine_inv3(m):
    """graph.cu inv3: the cofactor inverse of the 3x3 lattice (rows = lattice vectors) in the engine's operation order,
    so that fractional coordinates and heights derived from it are bit-identical to the engine's"""
    m = [float(v) for v in np.asarray(m, dtype=np.float64).reshape(9)]
    det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6])
    i = 1.0 / det
    o = [(m[4] * m[8] - m[5] * m[7]) * i, (m[2] * m[7] - m[1] * m[8]) * i, (m[1] * m[5] - m[2] * m[4]) * i,
         (m[5] * m[6] - m[3] * m[8]) * i, (m[0] * m[8] - m[2] * m[6]) * i, (m[2] * m[3] - m[0] * m[5]) * i,
         (m[3] * m[7] - m[4] * m[6]) * i, (m[1] * m[6] - m[0] * m[7]) * i, (m[0] * m[4] - m[1] * m[3]) * i]
    return np.array(o).reshape(3, 3)


def engine_wrap(cart, lattice, pbc):
    """graph.cu k_wrap: wrapped fractional coordinates, bit-identical to the engine's (separately rounded products and
    sums in the same order, exact fmod)"""
    cart = np.asarray(cart, dtype=np.float64)
    inv = engine_inv3(lattice)
    f = np.zeros_like(cart)
    for j in range(3):
        f[:, j] = ((0.0 + cart[:, 0] * inv[0, j]) + cart[:, 1] * inv[1, j]) + cart[:, 2] * inv[2, j]
        if pbc[j]:
            t = np.fmod(f[:, j], 1.0)
            t[t < 0] += 1.0
            f[:, j] = t
    return f


def axis_height(lattice, axis):
    """the cell's height across the lattice planes of `axis` (1 / |column axis of inv|), as graph.cu computes it"""
    inv = engine_inv3(lattice)
    return 1.0 / np.sqrt(inv[0, axis] * inv[0, axis] + inv[1, axis] * inv[1, axis] + inv[2, axis] * inv[2, axis])


def work_weights(i1, bond, n):
    """w_i = deg_i + nb_i (nb_i - 1): edges into atom i (the edges its owner processes) plus the angles centred on it;
    from neighbor_list's centre index i1 and bond mask (all False without a bond graph)"""
    deg = np.bincount(np.asarray(i1), minlength=n).astype(np.int64)
    nb = np.bincount(np.asarray(i1)[np.asarray(bond, dtype=bool)], minlength=n).astype(np.int64)
    return deg + nb * (nb - 1)


def balanced_walls(frac_axis, weights, P, delta, lo, hi):
    """graph.cu balanced policy: the P - 1 walls along the axis.

    Atoms sorted by coordinate x with the inclusive prefix S of their integer weights; wall k (1..P-1) goes half-way
    between x[i], i the first atom with S[i] P >= k S[-1], and the next larger coordinate (the next smaller when x[i]
    is the largest).  Then every slab is widened to delta: forward w_k >= w_(k-1) + delta, backward
    w_k <= w_(k+1) - delta, with w_(-1) = lo and w_(P-1) = hi.  Raises SlabWidthError when a slab is still thinner than
    delta (relative slack 1e-12 for the rounding of the passes).  Last the collision nudge of partition_rule."""
    x = np.asarray(frac_axis, dtype=np.float64)
    order = np.argsort(x, kind="stable")
    xs = x[order]
    S = np.cumsum(np.asarray(weights, dtype=np.int64)[order])
    n = len(xs)
    walls = []
    for k in range(1, P):
        i = int(np.argmax(S * P >= k * S[-1]))
        j = int(np.searchsorted(xs, xs[i], side="right"))
        if j < n:
            a, b = xs[i], xs[j]
        else:
            lft = int(np.searchsorted(xs, xs[i], side="left"))
            a, b = (xs[lft - 1] if lft > 0 else xs[i]), xs[i]
        walls.append(0.5 * (float(a) + float(b)))
    for k in range(P - 1):
        walls[k] = max(walls[k], (walls[k - 1] if k else lo) + delta)
    for k in range(P - 2, -1, -1):
        walls[k] = min(walls[k], (walls[k + 1] if k + 1 < P - 1 else hi) - delta)
    for k in range(P):
        width = (walls[k] if k < P - 1 else hi) - (walls[k - 1] if k else lo)
        if width < delta * (1 - 1e-12):
            raise SlabWidthError(k, width, delta)
    walls = np.array(walls, dtype=np.float64)
    for _ in range(64):
        hit = np.array([np.any(x == w) for w in walls], dtype=bool)
        if not hit.any():
            break
        walls[hit] += EPSILON
    return walls


def balanced_partition(frac_wrapped, lattice, pbc, P, cutoff, bond_cutoff, weights, walls_from_min=False):
    """(axis, walls) of the engine's balanced policy for the engine's wrapped fractional coordinates (engine_wrap):
    axis of the longest Cartesian extent, end bounds 0 and 1 on a periodic axis and the lowest / highest atom otherwise
    (or for an unfolded heat-flux cell), delta = 2 (cutoff + bond_cutoff) / height.  Raises SlabWidthError (with width
    and need in Angstrom) when infeasible."""
    lattice = np.asarray(lattice, dtype=np.float64)
    ext = (frac_wrapped @ lattice).max(axis=0) - (frac_wrapped @ lattice).min(axis=0)
    dim = 0
    for i in (1, 2):
        if ext[i] > ext[dim]:
            dim = i
    f = frac_wrapped[:, dim]
    from_min = walls_from_min or not pbc[dim]
    lo, hi = (float(f.min()), float(f.max())) if from_min else (0.0, 1.0)
    need = 2 * (cutoff + bond_cutoff)
    h = axis_height(lattice, dim)
    try:
        return dim, balanced_walls(f, weights, P, need / h, lo, hi)
    except SlabWidthError as e:
        raise SlabWidthError(e.slab, e.width * h, need) from None


class WalledOracle(GraphOracle):
    """GraphOracle of the partition given by `axis` and `walls` (e.g. balanced_partition's) instead of the reference's
    equally spaced walls: the same neighbour list, owners = number of walls <= coordinate, to / from lists from them."""

    def __init__(self, cart, lattice, pbc, axis, walls, cutoff, bond_cutoff, use_bond_graph=True, tol=1e-8,
                 frac_wrapped=None):
        super().__init__(cart, lattice, pbc, 1, cutoff, bond_cutoff, use_bond_graph, tol, frac_wrapped)
        self.P = len(walls) + 1
        self.dim, self.walls = axis, np.asarray(walls, dtype=np.float64)
        self.owner = which_partition(self.frac[:, axis], self.walls)
        self.accepts = True
        src, dst = self.i1, self.i2
        cross = self.owner[src] != self.owner[dst]
        self.to_part = np.full(self.n, -1, dtype=np.int64)
        self.to_part[src[cross]] = self.owner[dst[cross]]
        pairs = np.unique(np.column_stack([src[cross], self.owner[dst[cross]]]), axis=0)
        self.unique_to = len(np.unique(pairs[:, 0])) == len(pairs)  # one "to" partition per atom
