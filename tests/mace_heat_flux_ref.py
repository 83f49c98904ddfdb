"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Heat flux of MACE in the unfolded-cell form of oracle/heat_flux_ref.py (DESIGN.md §10): the same definitions and the
same `unfold`, CPU, float64, by autograd over `node_energies`, which the three MACE restatements share (oracle/mace_ref.py,
tests/mace_eq_ref.py, tests/mace_zbl_ref.py).  What differs from CHGNet and TensorNet:

  reach  T r_max: h[0] depends on the species only, each of the T interactions adds one r_max hop (the readout of layer
         t sees t + 1 of them), the ZBL pair term is one hop and the Agnesi transform acts on one edge
  U_j    eps_j, the per-atom energy with E0, scale and shift included (MACE has no data_mean), so J_conv = sum_{i<n} U_i v_i
  species mace_ref.species_index; the naive flux -sum_i w_i v_i from mace_ref.atomic_virials_ref

`mutants=True` gives the J_pot of the three bugs of oracle/heat_flux_ref.py and of two MACE-specific ones, in which a
term the engine differentiates outside the readout seeds keeps weight 1 on every unfolded atom instead of its readout
weight (the cell mask or the position seed):
  zbl_unweighted             the ZBL force term scale dV_e/dd of k_mace_edge_final (the pair energy of edge e belongs to
                             dst(e)); only for a model with pair repulsion
  readout_adjoint_unweighted the adjoint of the linear readouts of layers 0 .. T - 2 (k_mace_add_row)
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.heat_flux_ref import unfold
from oracle.mace_ref import atomic_virials_ref, species_index


def reach_of(model):
    """receptive-field radius of a MACE atom's energy: num_interactions * r_max"""
    return len(model.interactions) * float(model.r_max)


class UnfoldedModel:
    """Per-atom energies U_j of every unfolded atom as a function of the unfolded positions, on the fixed r_max
    neighbour list of the given positions (no periodicity)."""

    def __init__(self, model, ucart, lattice, z, dtype=torch.float64):
        from oracle.graph_ref import neighbor_list

        self.model = model.to(dtype)
        i1, i2, _off, _d2, _b = neighbor_list(ucart, lattice, np.zeros(3, dtype=np.int64), float(model.r_max), 0.0)
        t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int64)  # noqa: E731
        self.src, self.dst, self.z = t(i1), t(i2), t(z)
        self.n_edges = len(i1)

    def energies(self, pos):
        return self.model.node_energies(pos[self.dst] - pos[self.src], self.src, self.dst, self.z)[0]

    def energies_and_parts(self, pos):
        """(U, L, P) [N]: U, and the parts of it that the linear readouts (L) and the ZBL pair term (P) contribute, all
        in the autograd graph (forward hooks on those modules; zero where the model has none)"""
        m, out, hooks = self.model, {"lin": [], "pair": []}, []
        for ro in list(m.readouts)[:-1]:
            hooks.append(ro.register_forward_hook(lambda _m, _i, o: out["lin"].append(o)))
        if getattr(m, "pair_repulsion", False):
            hooks.append(m.pair_repulsion_fn.register_forward_hook(lambda _m, _i, o: out["pair"].append(o)))
        try:
            U = self.energies(pos)
        finally:
            for h in hooks:
                h.remove()
        s = m.scale_shift.scale
        return U, s * sum(out["lin"], torch.zeros_like(U)), s * sum(out["pair"], torch.zeros_like(U))


def heat_flux_ref(model, atoms, velocities, reach=None, centre=None, dtype=torch.float64, jacobian=False, naive=False,
                  mutants=False):
    """dict of numpy arrays with the keys of oracle/heat_flux_ref.py heat_flux_ref: j_pot [3], j_conv [3], energy,
    forces [n,3] (folded), energies [n] (cell eps_i), forces_unfolded [N,3] (F~), n_unfolded, n_edges, image_of,
    unfolded, G, centre, scale; with jacobian=True j_pot_def [3]; with naive=True j_naive [3]; with mutants=True the
    J_pot of the bugs above (dict)."""
    lattice = np.array(atoms.get_cell(), dtype=np.float64)
    cart = np.array(atoms.get_positions(), dtype=np.float64)
    n = len(cart)
    v = np.asarray(velocities, dtype=np.float64).reshape(n, 3)
    reach = reach_of(model) if reach is None else float(reach)
    ucart, image_of = unfold(cart, lattice, atoms.get_pbc().astype(np.int64), reach)
    N = len(ucart)
    um = UnfoldedModel(model, ucart, lattice, species_index(model, atoms).numpy()[image_of], dtype)
    c = 0.5 * lattice.sum(0) if centre is None else np.asarray(centre, dtype=np.float64)
    pos = torch.tensor(ucart, dtype=dtype, requires_grad=True)
    U, L, P = um.energies_and_parts(pos)
    rc = ucart - c
    cell = np.where(np.arange(N) < n, 1.0, 0.0)
    seeds = [cell * rc[:, a] for a in range(3)]

    def grad(w, X):
        (g,) = torch.autograd.grad((torch.as_tensor(w, dtype=dtype) * X).sum(), pos, retain_graph=True, allow_unused=True)
        return np.zeros((N, 3)) if g is None else g.numpy()

    vu = v[image_of]

    def j_pot_of(G, Ft, r=rc):
        fv = np.einsum("jk,jk->j", Ft, vu)
        return np.array([np.einsum("jk,jk->", G[a], vu) + (r[:, a] * fv).sum() for a in range(3)])

    Ft = -grad(cell, U)
    G = [grad(seeds[a], U) for a in range(3)]
    j_pot = j_pot_of(G, Ft)
    fv = np.einsum("jk,jk->j", Ft, vu)
    # size of the sum's terms: what an fp32 evaluation's round-off is relative to
    scale = max(np.abs(np.einsum("jk,jk->j", G[a], vu)).sum() + np.abs(rc[:, a] * fv).sum() for a in range(3))
    eps = U.detach()[:n]
    out = dict(j_pot=j_pot, j_conv=(eps.numpy()[:, None] * v).sum(0), energy=float(eps.sum()), energies=eps.numpy(),
               forces=np.zeros((n, 3)), forces_unfolded=Ft, n_unfolded=N, n_edges=um.n_edges, image_of=image_of,
               unfolded=ucart, G=np.stack(G), centre=c, scale=scale)
    np.add.at(out["forces"], image_of, Ft)
    if jacobian:
        jac = torch.autograd.functional.jacobian(lambda p: um.energies(p)[:n], pos.detach())  # [n, N, 3]
        dUv = np.einsum("ijk,jk->ij", jac.numpy(), vu)  # dU_i/dr_j . v_j
        rij = ucart[:n, None, :] - ucart[None, :, :]
        out["j_pot_def"] = np.einsum("ija,ij->a", rij, dUv)
    if naive:
        w = atomic_virials_ref(model, atoms, dtype).numpy()
        out["j_naive"] = -np.einsum("iab,ib->a", w, v)
    if mutants:
        ones = np.ones(N)
        m = {"images_dropped": np.array([np.einsum("jk,jk->", G[a][:n], vu[:n]) + (rc[:n, a] * fv[:n]).sum()
                                         for a in range(3)]),
             "seed_unmasked": j_pot_of([grad(rc[:, a], U) for a in range(3)], Ft),
             "centre_in_one_term": j_pot_of(G, Ft, ucart)}

        def unweighted(X):  # the part X of U differentiated with weight 1 instead of the mask and the seeds
            gx = grad(ones, X)
            return j_pot_of([G[a] - grad(seeds[a], X) + gx for a in range(3)], Ft + grad(cell, X) - gx)

        if getattr(model, "pair_repulsion", False):
            m["zbl_unweighted"] = unweighted(P)
        if len(model.readouts) > 1:
            m["readout_adjoint_unweighted"] = unweighted(L)
        out["mutants"] = m
    return out


def barycentre(model, atoms, velocities, t, reach=None, dtype=torch.float64):
    """B(t) = sum_{i<n} r_i(t) U_i(r(t)) with every unfolded atom moved along r + t v (v of the atom it images), and
    the neighbour list of t = 0 (the envelopes make the energy smooth across it)"""
    lattice = np.array(atoms.get_cell(), dtype=np.float64)
    cart = np.array(atoms.get_positions(), dtype=np.float64)
    n = len(cart)
    ucart, image_of = unfold(cart, lattice, atoms.get_pbc().astype(np.int64), reach_of(model) if reach is None else reach)
    um = UnfoldedModel(model, ucart, lattice, species_index(model, atoms).numpy()[image_of], dtype)
    vu = np.asarray(velocities, dtype=np.float64)[image_of]
    out = []
    with torch.no_grad():
        for tt in t:
            p = torch.tensor(ucart + tt * vu, dtype=dtype)
            out.append((p[:n] * um.energies(p)[:n, None]).sum(0).numpy())
    return np.array(out)
