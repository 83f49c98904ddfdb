"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Per-atom energies and per-atom virials of CHGNet and TensorNet by autograd over the global graph, for the engine's
`b2m_get_atomic` (DESIGN.md "Per-atom energies and virials").  Reuses `forward_graph` of oracle/chgnet_ref.py and
oracle/tensornet_ref.py; the geometry is that of their `potential_ref` (pes.py:50-146), with the edge vectors kept as a
leaf of the graph so that autograd yields g_e = dE/dv_e.

  eps_i = data_std * e_atom_i + element_ref[Z_i] + data_mean / N          (sums to E)
  w_i   = 1/2 sum_{e : i in {src_e, dst_e}} v_e (x) g_e                     (sums to the strain derivative of E)
"""
from __future__ import annotations

import numpy as np
import torch

GPA_PER_EV_A3 = 160.21766208


def atomic_ref(model, atoms, data_mean=0.0, data_std=1.0, element_refs=None, dtype=torch.float64, edges=False):
    """Returns a dict of torch tensors: energies [N], virials [N,3,3] (eV), energy (scalar), strain_virial [3,3]
    (dE/d strain, eV), stress [3,3] (GPa), forces [N,3].  With `edges=True` also the per-edge parts the virials are
    made of, in the neighbour list's order: edge_src [E], edge_dst [E], edge_off [E,3] (int64 image of dst) and
    edge_half [E,3,3] = 1/2 v_e (x) g_e, which goes once to each endpoint."""
    from oracle.graph_ref import neighbor_list

    tensornet = hasattr(model, "tensor_embedding")
    lattice_np = np.array(atoms.get_cell())
    cart = np.array(atoms.get_positions(wrap=False))
    pbc = atoms.get_pbc().astype(np.int64)
    rb = 0.0 if tensornet else float(model.three_body_cutoff)
    i1, i2, off, _d2, bond = neighbor_list(cart, lattice_np, pbc, float(model.cutoff), rb)
    model = model.to(dtype)
    strain = torch.zeros(3, 3, dtype=dtype, requires_grad=True)
    lattice = torch.tensor(lattice_np, dtype=dtype) @ (torch.eye(3, dtype=dtype) + strain)
    pos = torch.tensor(atoms.get_scaled_positions(False), dtype=dtype) @ lattice
    pos.retain_grad()
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int64)
    src, dst = t(i1), t(i2)
    vec = pos[dst] + torch.tensor(off, dtype=dtype) @ lattice - pos[src]
    vec.retain_grad()
    el2idx = {el: k for k, el in enumerate(model.element_types)}
    node_types = t([el2idx[s] for s in atoms.get_chemical_symbols()])
    taps = {}
    if tensornet:
        e_raw = model.forward_graph(vec, src, dst, node_types, taps=taps)
    else:
        from oracle.chgnet_ref import build_line_graph

        bond_edges, la, lb, ce = build_line_graph(i1, i2, bond)
        e_raw, _site = model.forward_graph(pos, vec, src, dst, t(bond_edges), t(la), t(lb), t(ce), node_types,
                                           taps=taps)
    n = len(atoms)
    eps = data_std * taps["e_atom"].detach().reshape(n).to(dtype) + data_mean / n
    total = data_std * e_raw + data_mean
    if element_refs is not None:
        ref = torch.as_tensor(np.asarray(element_refs), dtype=dtype)[node_types]
        eps = eps + ref
        total = total + ref.sum()
    total.backward()
    g = vec.grad
    half = 0.5 * vec.detach()[:, :, None] * g[:, None, :]  # [E,3,3]: 1/2 v_e (x) g_e
    vir = torch.zeros(n, 3, 3, dtype=dtype).index_add_(0, src, half).index_add_(0, dst, half)
    vol = abs(np.linalg.det(lattice_np))
    out = dict(energies=eps, virials=vir, energy=total.detach(), strain_virial=strain.grad.detach(),
               stress=strain.grad.detach() / vol * GPA_PER_EV_A3, forces=-pos.grad.detach())
    if edges:
        out.update(edge_src=src, edge_dst=dst, edge_off=t(off), edge_half=half)
    return out


def routing_mutants(src, dst, half, n, order=None):
    """Per-atom virials [N,3,3] of plausible routing bugs of a kernel that walks the edges in `order` (default: sorted
    by destination, stably) one edge per lane, 32 lanes per warp, and adds the destination halves once per run of
    equal destinations.  Returns {name: virials}; "next atom" is the destination of the following run (cyclically).

      last_edge_to_next   the last edge of every run adds its destination half to the next atom
      run_to_next         every run adds its destination halves to the next atom
      all_to_dst          the source half goes to the destination as well
      src_transposed      the source receives (1/2 v (x) g)^T
      straddle_to_next    a run cut by a multiple of 32: the part before the last cut goes to the next atom
    """
    src, dst = torch.as_tensor(src), torch.as_tensor(dst)
    if order is None:
        order = torch.argsort(dst, stable=True)
    order = torch.as_tensor(order)
    s, d, h = src[order], dst[order], half[order]
    E = len(d)
    pos = torch.arange(E)
    start = torch.ones(E, dtype=torch.bool)
    start[1:] = d[1:] != d[:-1]
    end = torch.ones(E, dtype=torch.bool)
    end[:-1] = start[1:]
    run = torch.cumsum(start.long(), 0) - 1
    next_atom = d[start].roll(-1)[run]  # per edge: the destination of the following run
    last = pos[end][run]                # per edge: position of its run's last edge
    z = lambda: torch.zeros(n, 3, 3, dtype=h.dtype)
    src_part = z().index_add_(0, s, h)

    def with_dst(target):
        return src_part + z().index_add_(0, target, h)

    return {
        "last_edge_to_next": with_dst(torch.where(pos == last, next_atom, d)),
        "run_to_next": with_dst(next_atom),
        "all_to_dst": z().index_add_(0, d, 2 * h),
        "src_transposed": z().index_add_(0, s, h.transpose(1, 2)) + z().index_add_(0, d, h),
        "straddle_to_next": with_dst(torch.where(pos // 32 < last // 32, next_atom, d)),
    }
