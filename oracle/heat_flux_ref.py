"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Heat flux of CHGNet and TensorNet in the unfolded-cell form (DESIGN.md §10; Langer, Frank, Knoop, Phys. Rev. B 108,
L100302 (2023)), CPU, float64, by autograd over the `forward_graph`s that oracle/atomic_ref.py uses.

  unfolded cell: the n cell atoms, then every periodic image j + s.L within `reach` of them (periodic axes only), with
                 image_of[j'] = j; evaluated without periodicity; U = sum_{i<n} U_i
  J_pot^a  = sum_j [ G^a_j . v_j + (r_j - c)_a (F~_j . v_j) ],   G^a_j = sum_{i<n} (r_i - c)_a dU_i/dr_j,  F~ = -dU/dr
  J_conv   = sum_{i<n} eps_i v_i      (eps_i: the per-atom energies of atomic_ref, data_mean / n and element refs included)

`heat_flux_ref(..., jacobian=True)` also returns the definition sum_{i<n} sum_j r_ij (dU_i/dr_j . v_j) from the full
Jacobian (tiny cells only), and `naive=True` the edge-split virial flux -sum_i w_i v_i of the periodic per-atom virials.
"""
from __future__ import annotations

import numpy as np
import torch


def reach_of(model):
    """receptive-field radius of an atom's energy: CHGNet max(n_blocks r_cut, r_cut + (n_blocks - 1) r_bond), TensorNet
    (nblocks + 1) r_cut"""
    if hasattr(model, "tensor_embedding"):
        return (int(model.nblocks) + 1) * float(model.cutoff)
    nb, rc, rb = int(model.n_blocks), float(model.cutoff), float(model.three_body_cutoff)
    return max(nb * rc, rc + (nb - 1) * rb)


def unfold(cart, lattice, pbc, reach):
    """(unfolded positions [N,3], image_of [N]): the cell atoms, then for every atom (in order) its images with shift s
    in lexicographic order, admitted when every periodic fractional coordinate lies in the cell atoms' fractional
    bounding box widened by reach / h_k (h_k: height of the cell across lattice plane k)"""
    cart = np.asarray(cart, dtype=np.float64)
    lattice = np.asarray(lattice, dtype=np.float64)
    inv = np.linalg.inv(lattice)
    frac = cart @ inv
    n = len(cart)
    lo, hi = frac.min(0), frac.max(0)
    ranges = []
    for k in range(3):
        if pbc[k]:
            pad = reach * np.linalg.norm(inv[:, k])
            lo[k], hi[k] = lo[k] - pad, hi[k] + pad
            ranges.append(range(int(np.ceil(lo[k] - frac[:, k].max())), int(np.floor(hi[k] - frac[:, k].min())) + 1))
        else:
            ranges.append(range(0, 1))
    shifts = np.array([(a, b, c) for a in ranges[0] for b in ranges[1] for c in ranges[2] if (a, b, c) != (0, 0, 0)],
                      dtype=np.float64).reshape(-1, 3)
    g = frac[:, None, :] + shifts[None, :, :]  # [n, S, 3]
    ok = np.ones(g.shape[:2], dtype=bool)
    for k in range(3):
        if pbc[k]:
            ok &= (g[:, :, k] >= lo[k]) & (g[:, :, k] <= hi[k])
    ii, ss = np.nonzero(ok)  # atom-major, shifts in lexicographic order
    images = cart[ii] + shifts[ss] @ lattice
    return np.concatenate([cart, images]), np.concatenate([np.arange(n), ii]).astype(np.int64)


class UnfoldedModel:
    """Per-atom energies U_j (data_std * e_atom_j; constants left out) of every unfolded atom as a function of the
    unfolded positions, on the fixed neighbour list of the given positions (no periodicity)."""

    def __init__(self, model, ucart, lattice, node_types, data_std=1.0, dtype=torch.float64):
        from oracle.graph_ref import neighbor_list

        self.tensornet = hasattr(model, "tensor_embedding")
        self.model = model.to(dtype)
        self.dtype, self.data_std = dtype, data_std
        rb = 0.0 if self.tensornet else float(model.three_body_cutoff)
        i1, i2, _off, _d2, bond = neighbor_list(ucart, lattice, np.zeros(3, dtype=np.int64), float(model.cutoff), rb)
        t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int64)
        self.src, self.dst, self.types = t(i1), t(i2), t(node_types)
        self.n_edges = len(i1)
        if not self.tensornet:
            from oracle.chgnet_ref import build_line_graph

            self.lg = [t(a) for a in build_line_graph(i1, i2, bond)]

    def energies(self, pos):
        vec = pos[self.dst] - pos[self.src]
        taps = {}
        if self.tensornet:
            # TensorNetRef.forward_graph with the per-atom energies kept in the autograd graph (its tap is detached)
            from oracle.tensornet_ref import decompose_tensor, tensor_norm

            m, src, dst = self.model, self.src, self.dst
            d = torch.linalg.norm(vec, dim=1)
            edge_attr = m.bond_expansion(d)
            X = m.tensor_embedding(src, dst, self.types, d, vec, edge_attr, len(self.types))
            for layer in m.layers:
                X = layer(src, dst, d, edge_attr, X)
            I, A, S = decompose_tensor(X)
            x = m.linear(m.out_norm(torch.cat((tensor_norm(I), tensor_norm(A), tensor_norm(S)), dim=-1)))
            return self.data_std * m.final_layer.gated(x).reshape(-1).to(self.dtype)
        else:
            self.model.forward_graph(pos, vec, self.src, self.dst, *self.lg, self.types, taps=taps)
        return self.data_std * taps["e_atom"].reshape(-1).to(self.dtype)


def heat_flux_ref(model, atoms, velocities, reach=None, data_mean=0.0, data_std=1.0, element_refs=None, centre=None,
                  dtype=torch.float64, jacobian=False, naive=False, mutants=False):
    """dict of numpy arrays: j_pot [3], j_conv [3], energy, forces [n,3] (folded), energies [n] (cell eps_i),
    forces_unfolded [N,3] (F~), n_unfolded, n_edges; with jacobian=True j_pot_def [3]; with naive=True j_naive [3]
    (-sum_i w_i v_i, periodic edge-split virials); with mutants=True the J_pot of four plausible bugs (dict)."""
    lattice = np.array(atoms.get_cell(), dtype=np.float64)
    cart = np.array(atoms.get_positions(), dtype=np.float64)
    pbc = atoms.get_pbc().astype(np.int64)
    n = len(cart)
    v = np.asarray(velocities, dtype=np.float64).reshape(n, 3)
    reach = reach_of(model) if reach is None else float(reach)
    ucart, image_of = unfold(cart, lattice, pbc, reach)
    N = len(ucart)
    el2idx = {el: k for k, el in enumerate(model.element_types)}
    types = np.array([el2idx[s] for s in atoms.get_chemical_symbols()])
    um = UnfoldedModel(model, ucart, lattice, types[image_of], data_std, dtype)
    c = 0.5 * lattice.sum(0) if centre is None else np.asarray(centre, dtype=np.float64)
    pos = torch.tensor(ucart, dtype=dtype, requires_grad=True)
    U = um.energies(pos)
    cell = torch.zeros(N, dtype=dtype)
    cell[:n] = 1.0
    (g_mask,) = torch.autograd.grad((cell * U).sum(), pos, retain_graph=True)
    Ft = -g_mask.detach().numpy()  # F~
    rc = ucart - c
    G = []
    for a in range(3):
        seed = torch.tensor(np.where(np.arange(N) < n, rc[:, a], 0.0), dtype=dtype)
        (g,) = torch.autograd.grad((seed * U).sum(), pos, retain_graph=True)
        G.append(g.numpy())
    vu = v[image_of]
    fv = np.einsum("jk,jk->j", Ft, vu)
    j_pot = np.array([np.einsum("jk,jk->", G[a], vu) + (rc[:, a] * fv).sum() for a in range(3)])
    # size of the sum's terms: what an fp32 evaluation's round-off is relative to
    scale = max(np.abs(np.einsum("jk,jk->j", G[a], vu)).sum() + np.abs(rc[:, a] * fv).sum() for a in range(3))
    ref = torch.as_tensor(np.zeros(len(types)) if element_refs is None else np.asarray(element_refs)[types], dtype=dtype)
    eps = U.detach()[:n] + ref + data_mean / n
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
        from oracle.atomic_ref import atomic_ref

        w = atomic_ref(model, atoms, data_mean, data_std, element_refs, dtype)["virials"].numpy()
        out["j_naive"] = -np.einsum("iab,ib->a", w, v)
    if mutants:
        # the images' contributions dropped from the sums over j
        no_img = np.array([np.einsum("jk,jk->", G[a][:n], vu[:n]) + (rc[:n, a] * fv[:n]).sum() for a in range(3)])
        # the seed not masked on the images: sum over all unfolded atoms of (r_i - c)_a U_i
        G_all = []
        for a in range(3):
            (g,) = torch.autograd.grad((torch.tensor(rc[:, a], dtype=dtype) * U).sum(), pos, retain_graph=True)
            G_all.append(g.numpy())
        unmasked = np.array([np.einsum("jk,jk->", G_all[a], vu) + (rc[:, a] * fv).sum() for a in range(3)])
        # c applied to the seed only: (r_j)_a in the second term
        one_c = np.array([np.einsum("jk,jk->", G[a], vu) + (ucart[:, a] * fv).sum() for a in range(3)])
        out["mutants"] = {"images_dropped": no_img, "seed_unmasked": unmasked, "centre_in_one_term": one_c}
    return out


def barycentre(model, atoms, velocities, t, reach=None, data_std=1.0, dtype=torch.float64):
    """B(t) = sum_{i<n} r_i(t) U_i(r(t)) with every unfolded atom moved along r + t v (v of the atom it images), and
    the neighbour list of t = 0 (the envelopes make the energy smooth across it)"""
    lattice = np.array(atoms.get_cell(), dtype=np.float64)
    cart = np.array(atoms.get_positions(), dtype=np.float64)
    n = len(cart)
    ucart, image_of = unfold(cart, lattice, atoms.get_pbc().astype(np.int64), reach_of(model) if reach is None else reach)
    el2idx = {el: k for k, el in enumerate(model.element_types)}
    types = np.array([el2idx[s] for s in atoms.get_chemical_symbols()])
    um = UnfoldedModel(model, ucart, lattice, types[image_of], data_std, dtype)
    vu = np.asarray(velocities, dtype=np.float64)[image_of]
    out = []
    with torch.no_grad():
        for tt in t:
            p = torch.tensor(ucart + tt * vu, dtype=dtype)
            out.append((p[:n] * um.energies(p)[:n, None]).sum(0).numpy())
    return np.array(out)
