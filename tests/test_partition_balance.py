"""Work-balanced slab partitions (DESIGN.md §4.1) on the CPU: the restatement tests/balance_ref.balanced_walls on a
hand-worked case, and the balance it reaches on non-uniform cells against the reference's equally spaced walls.

The structure builders here are shared with tests/test_gpu_partition_balance.py and tests/balance_times.py.
"""
import numpy as np
import pytest

from distmlip_b200.structures import SI_A, SimpleAtoms, si_diamond
from oracle import graph_ref as G
from tests import balance_ref as B

_DIAMOND_BASIS = np.array([[0, 0, 0], [0, .5, .5], [.5, 0, .5], [.5, .5, 0],
                           [.25, .25, .25], [.25, .75, .75], [.75, .25, .75], [.75, .75, .25]])
RC, RB = 5.0, 3.0  # CHGNet's cutoffs: slabs at least 2 (RC + RB) = 16 A wide


def _diamond_frac(n, nz, sigma, rng):
    """unwrapped diamond sites of an n x n x nz block in units of the conventional cell, perturbed"""
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
    f = (g[:, None, :] + _DIAMOND_BASIS[None]).reshape(-1, 3).astype(np.float64)
    return f + rng.normal(0.0, sigma / SI_A, size=f.shape)


def _gas(count, lo, hi, min_dist, rng, periodic_box):
    """`count` random points in the box [lo, hi), none closer than min_dist to another (later ones of a close pair are
    dropped, then the box is topped up)"""
    from scipy.spatial import cKDTree

    pts = np.zeros((0, 3))
    for _ in range(50):
        if len(pts) >= count:
            break
        cand = np.concatenate([pts, lo + rng.random((2 * (count - len(pts)) + 8, 3)) * (hi - lo)])
        t = cKDTree(np.mod(cand, periodic_box), boxsize=periodic_box)
        bad = {j for i, j in t.query_pairs(min_dist)}  # i < j: keep the earlier point
        pts = cand[[k for k in range(len(cand)) if k not in bad]]
    return pts[:count]


def two_phase(n, nz, seed=0, sigma=0.15, gas_density=0.03):
    """perturbed diamond Si filling the lower half (nz conventional cells) of an n x n x 2 nz cell, a dilute gas of
    gas_density times the crystal's density in the upper half, gas atoms >= 2.2 A from each other and from the crystal"""
    rng = np.random.default_rng(seed)
    L = np.array([n * SI_A, n * SI_A, 2 * nz * SI_A])
    crystal = _diamond_frac(n, nz, sigma, rng) * SI_A
    ngas = int(round(gas_density * len(crystal)))
    gas = _gas(ngas, np.array([0.0, 0.0, nz * SI_A + 2.2]), np.array([L[0], L[1], L[2] - 2.2]), 2.2, rng,
               np.array([L[0], L[1], 4 * L[2]]))
    pos = np.concatenate([crystal, gas])
    return SimpleAtoms(["Si"] * len(pos), pos, np.diag(L))


def particle(radius, seed=0, sigma=0.15, vacuum=12.0, pbc=True):
    """a sphere cut from perturbed diamond Si, centred in a cubic box with `vacuum` Angstrom between periodic images"""
    rng = np.random.default_rng(seed)
    m = int(np.ceil(2 * radius / SI_A)) + 2
    pos = (_diamond_frac(m, m, sigma, rng) - m / 2) * SI_A
    pos = pos[np.einsum("ij,ij->i", pos, pos) <= radius * radius]
    box = 2 * radius + vacuum + 1.0
    pos = pos + box / 2
    return SimpleAtoms(["Si"] * len(pos), pos, np.eye(3) * box, pbc=(pbc, pbc, pbc))


def tilted(n=3, nz=6, seed=0):
    """the two-phase cell with its first lattice vector tilted out of the xy plane by t = n a: the lattice column of
    the partition axis grows to sqrt(t^2 + Lz^2) while the height across the walls shrinks to Lz Lx / sqrt(t^2 + Lx^2)
    (46.1 A here): at P = 3 the reference's column check passes (22.4 A > 16 A) but 3 slabs of 16 A do not fit"""
    a = two_phase(n, nz, seed=seed)
    lat = a.get_cell()
    frac = a.get_positions() @ np.linalg.inv(lat)
    lat[0, 2] = n * SI_A
    return SimpleAtoms(a.get_chemical_symbols(), frac @ lat, lat)


def uniform(n=4, nz=12, seed=3):
    return si_diamond(n, nz=nz, seed=seed)


def work_and_frac(atoms, rc=RC, rb=RB):
    """the engine's wrapped fractional coordinates and the graph_ref work of every atom"""
    cart, lat, pbc = atoms.get_positions(), atoms.get_cell(), atoms.get_pbc().astype(np.int64)
    i1, _i2, _off, _d2, bond = G.neighbor_list(cart, lat, pbc, rc, rb)
    return B.engine_wrap(cart, lat, pbc), B.work_weights(i1, bond, len(cart))


def imbalance(frac_axis, w, walls):
    """max / mean of the work per partition"""
    per = np.bincount(G.which_partition(frac_axis, walls), weights=w, minlength=len(walls) + 1)
    return per.max() / per.mean()


def equal_walls(atoms, frac, P):
    return G.partition_rule(frac @ atoms.get_cell(), frac, P)


# ---------------------------------------------------------------------------------------------------------------------
def test_hand_worked_case():
    x = np.array([0.02, 0.11, 0.13, 0.25, 0.31, 0.48, 0.52, 0.67, 0.81, 0.95])
    w = np.array([1, 5, 1, 2, 1, 3, 3, 1, 2, 1])  # prefix 1 6 7 9 10 13 16 17 19 20
    perm = np.random.default_rng(0).permutation(10)  # input order does not matter
    # P = 2: prefix first >= 10 at x = 0.31 -> half-way to 0.48
    assert B.balanced_walls(x[perm], w[perm], 2, 0.1, 0.0, 1.0).tolist() == [0.5 * (0.31 + 0.48)]
    # P = 4: prefix >= 5, 10, 15 at 0.11, 0.31, 0.52
    assert B.balanced_walls(x[perm], w[perm], 4, 0.1, 0.0, 1.0).tolist() == [
        0.5 * (0.11 + 0.13), 0.5 * (0.31 + 0.48), 0.5 * (0.52 + 0.67)]
    # P = 3 (prefix >= 20/3, 40/3 at 0.13, 0.52: walls 0.19, 0.595) with slabs >= 0.3: the forward pass moves both
    walls = B.balanced_walls(x[perm], w[perm], 3, 0.3, 0.0, 1.0)
    assert walls.tolist() == [0.3, 0.3 + 0.3]
    # the last wall when the quantile falls on the largest coordinate: the gap below it
    assert B.balanced_walls(np.array([0.1, 0.2, 0.9]), np.array([0, 0, 7]), 2, 0.0, 0.0, 1.0).tolist() == [0.55]


def test_every_slab_at_least_delta_wide():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.random(400) * 0.3, 0.3 + rng.random(20) * 0.7])  # dense third, sparse rest
    w = rng.integers(0, 60, size=len(x))
    for P, delta in [(2, 0.2), (4, 0.15), (6, 0.16), (8, 0.12)]:
        walls = B.balanced_walls(x, w, P, delta, 0.0, 1.0)
        edges = np.concatenate([[0.0], walls, [1.0]])
        assert np.all(np.diff(edges) >= delta * (1 - 1e-12)), (P, delta)
        assert not np.isin(walls, x).any()
    with pytest.raises(B.SlabWidthError) as ei:
        B.balanced_walls(x, w, 8, 0.13, 0.0, 1.0)  # 8 x 0.13 > 1
    assert 0 <= ei.value.slab < 8


@pytest.mark.parametrize("P", [2, 4])
def test_two_phase_balanced(P):
    atoms = two_phase(4, 12, seed=1)  # 65 A of crystal: four 16 A slabs fit in it
    assert 1500 < len(atoms) < 5000
    frac, w = work_and_frac(atoms)
    dim, walls = B.balanced_partition(frac, atoms.get_cell(), [1, 1, 1], P, RC, RB, w)
    assert dim == 2 and imbalance(frac[:, dim], w, walls) <= 1.05
    dim_e, walls_e = equal_walls(atoms, frac, P)
    assert dim_e == 2 and imbalance(frac[:, dim], w, walls_e) >= 1.3


def test_two_phase_balanced_eight_partitions():
    atoms = two_phase(3, 24, seed=2)  # 130 A of crystal: eight 16 A slabs fit
    assert 1500 < len(atoms) < 5000
    frac, w = work_and_frac(atoms)
    dim, walls = B.balanced_partition(frac, atoms.get_cell(), [1, 1, 1], 8, RC, RB, w)
    assert imbalance(frac[:, dim], w, walls) <= 1.05
    assert imbalance(frac[:, dim], w, equal_walls(atoms, frac, 8)[1]) >= 1.3


@pytest.mark.parametrize("pbc", [True, False])
def test_particle(pbc):
    """a sphere: equal slabs hold very different volumes at P >= 4 (at P = 2 they split it evenly by symmetry)"""
    atoms = particle(24.0, seed=4, pbc=pbc)
    assert 2000 < len(atoms) < 5000
    rc = 4.0  # without a bond graph (TensorNet, MACE): 8 A slabs, so four of them fit in the sphere unconstrained
    frac, w = work_and_frac(atoms, rc=rc, rb=0.0)
    pb = atoms.get_pbc().astype(int)
    for P in (2, 4):
        dim, walls = B.balanced_partition(frac, atoms.get_cell(), pb, P, rc, 0.0, w)
        assert imbalance(frac[:, dim], w, walls) <= 1.05, P
    for P in (4, 8):
        dim_e, walls_e = equal_walls(atoms, frac, P)
        assert imbalance(frac[:, dim_e], w, walls_e) >= 1.3, P


def test_where_the_width_binds_slabs_stay_wide():
    """two-phase cell with 65 A of crystal at P = 8, and the CHGNet particle: the width constraint binds; every slab is
    still >= 16 A across the walls; the balance is reported, not asserted"""
    for atoms, P in [(two_phase(4, 12, seed=1), 8), (particle(24.0, seed=4), 3)]:
        frac, w = work_and_frac(atoms)
        lat = atoms.get_cell()
        dim, walls = B.balanced_partition(frac, lat, [1, 1, 1], P, RC, RB, w)
        h = B.axis_height(lat, dim)
        edges = np.concatenate([[0.0], walls, [1.0]])
        assert np.all(np.diff(edges) * h >= 2 * (RC + RB) * (1 - 1e-9))
        bal = imbalance(frac[:, dim], w, walls)
        eq = imbalance(frac[:, dim], w, equal_walls(atoms, frac, P)[1])
        print(f"P={P}: max/mean balanced {bal:.3f}, equal {eq:.3f}")


def test_infeasible_width_is_detected():
    atoms = two_phase(3, 6, seed=0)  # Lz = 65 A: four 16 A slabs fit, five do not
    frac, w = work_and_frac(atoms)
    B.balanced_partition(frac, atoms.get_cell(), [1, 1, 1], 4, RC, RB, w)
    with pytest.raises(B.SlabWidthError) as ei:
        B.balanced_partition(frac, atoms.get_cell(), [1, 1, 1], 5, RC, RB, w)
    assert ei.value.need == 16.0 and ei.value.width < 16.0


def test_tilted_cell_uses_the_height():
    atoms = tilted()
    lat = atoms.get_cell()
    frac, w = work_and_frac(atoms)
    o = G.GraphOracle(atoms.get_positions(), lat, np.array([1, 1, 1]), 3, RC, RB, True, frac_wrapped=frac)
    assert o.dim == 2 and o.accepts  # the lattice column is long enough for three slabs
    with pytest.raises(B.SlabWidthError):
        B.balanced_partition(frac, lat, [1, 1, 1], 3, RC, RB, w)
    B.balanced_partition(frac, lat, [1, 1, 1], 2, RC, RB, w)


def test_engine_wrap_matches_wrap_frac():
    """the bit-exact restatement of k_wrap agrees with the reference restatement to round-off"""
    atoms = tilted()
    f1 = B.engine_wrap(atoms.get_positions(), atoms.get_cell(), [1, 1, 1])
    f2, _ = G.wrap_frac(atoms.get_positions(), atoms.get_cell(), [1, 1, 1])
    d = np.abs(f1 - f2)
    assert np.minimum(d, 1 - d).max() < 1e-12


def test_walled_oracle_with_the_reference_walls_is_the_reference_oracle():
    atoms = two_phase(3, 6, seed=0)
    cart, lat, pbc = atoms.get_positions(), atoms.get_cell(), np.array([1, 1, 1])
    frac = B.engine_wrap(cart, lat, pbc)
    o = G.GraphOracle(cart, lat, pbc, 3, RC, RB, True, frac_wrapped=frac)
    w = B.WalledOracle(cart, lat, pbc, o.dim, o.walls, RC, RB, True, frac_wrapped=frac)
    assert w.P == 3 and np.array_equal(w.owner, o.owner) and np.array_equal(w.to_part, o.to_part)
    assert w.unique_to == o.unique_to
    for p in range(3):
        assert np.array_equal(np.concatenate(w.edges_of(p)[:2]), np.concatenate(o.edges_of(p)[:2]))
        assert np.array_equal(w.angles_of(p), o.angles_of(p))
