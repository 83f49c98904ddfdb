"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Pure-PyTorch (CPU) restatement of the arithmetic behind the reference's CHGNet hot path:

  control flow / DistMLIP-specific behaviour .... DistMLIP/implementations/matgl/models/chgnet.py:21-453
                                                 DistMLIP/implementations/matgl/models/chgnet_layers.py:16-119
                                                 DistMLIP/implementations/matgl/pes.py:50-146
                                                 DistMLIP/distributed/dist.py:277-358, 635-702
  layer internals ............................... matgl @ git 5171392 (pyproject.toml:26-28), NOT in
                                                 the reference repository and not installed with it:
                                                 restated from SURVEY.md §9 "(RECALLED-matgl)".

PARITY UNPINNED: the reference ships no tests / golden vectors for the model arithmetic and
matgl+dgl are not available to the tests, so nothing in this file has been checked against a
run of the real reference.  What *is* pinned: the graph side (oracle/graph_ref.py vs oracle/_ref).

The module's attribute tree and state_dict keys mirror matgl's `CHGNet` (SURVEY.md §8c) so that
`CHGNet_Dist.from_existing` accepts either a real matgl model or this one.

Because the dist path's arithmetic is partition-independent (every `*_transfer` is a copy), one
evaluation over the global graph is the oracle for every partition count.
"""
from __future__ import annotations

import math

import numpy as np
import torch
from torch import nn

DEFAULT_ELEMENTS = (
    "H", "He", "Li", "Be", "B", "C", "N", "O", "F", "Ne", "Na", "Mg", "Al", "Si", "P", "S", "Cl", "Ar",
    "K", "Ca", "Sc", "Ti", "V", "Cr", "Mn", "Fe", "Co", "Ni", "Cu", "Zn", "Ga", "Ge", "As", "Se", "Br",
    "Kr", "Rb", "Sr", "Y", "Zr", "Nb", "Mo", "Tc", "Ru", "Rh", "Pd", "Ag", "Cd", "In", "Sn", "Sb", "Te",
    "I", "Xe", "Cs", "Ba", "La", "Ce", "Pr", "Nd", "Pm", "Sm", "Eu", "Gd", "Tb", "Dy", "Ho", "Er", "Tm",
    "Yb", "Lu", "Hf", "Ta", "W", "Re", "Os", "Ir", "Pt", "Au", "Hg", "Tl", "Pb", "Bi", "Ac", "Th", "Pa",
    "U", "Np", "Pu",
)


def polynomial_cutoff(r, cutoff, exponent):
    """matgl.utils.cutoff.polynomial_cutoff (RECALLED-matgl, SURVEY §9). NB: the reference
    feeds it the *rbf tensor*, not the distance (chgnet.py:116-124)."""
    coef1 = -(exponent + 1) * (exponent + 2) / 2
    coef2 = exponent * (exponent + 2)
    coef3 = -exponent * (exponent + 1) / 2
    ratio = r / cutoff
    env = 1 + coef1 * ratio**exponent + coef2 * ratio ** (exponent + 1) + coef3 * ratio ** (exponent + 2)
    return torch.where(r <= cutoff, env, torch.zeros_like(env))


class RadialBesselFunction(nn.Module):
    """(RECALLED-matgl) rbf_k(d) = sqrt(2/rc) sin(f_k d / rc) / d, f_k = k*pi learnable."""

    def __init__(self, max_n, cutoff, learnable=True):
        super().__init__()
        self.max_n = max_n
        self.cutoff = cutoff
        self.inv_cutoff = 1 / cutoff
        self.norm_const = (2 * self.inv_cutoff) ** 0.5
        freq = torch.pi * torch.arange(1, max_n + 1, dtype=torch.float32)
        if learnable:
            self.frequencies = nn.Parameter(freq)
        else:
            self.register_buffer("frequencies", freq)

    def forward(self, r):
        r = r[:, None]
        d_scaled = r * self.inv_cutoff
        return self.norm_const * torch.sin(self.frequencies * d_scaled) / r


class FourierExpansion(nn.Module):
    """(RECALLED-matgl) [cos(0), sin(f1 x), cos(f1 x), ...]/interval : even cols cos(k), odd cols sin(k>=1)."""

    def __init__(self, max_f=4, interval=math.pi, scale_factor=1.0, learnable=True):
        super().__init__()
        self.max_f = max_f
        self.interval = interval
        self.scale_factor = scale_factor
        freq = torch.arange(0, max_f + 1, dtype=torch.float32)
        if learnable:
            self.frequencies = nn.Parameter(freq)
        else:
            self.register_buffer("frequencies", freq)

    def forward(self, x):
        result = x.new_zeros(x.shape[0], 1 + 2 * self.max_f)
        tmp = torch.outer(x, self.frequencies)
        result[:, ::2] = torch.cos(tmp * math.pi / self.interval)
        result[:, 1::2] = torch.sin(tmp[:, 1:] * math.pi / self.interval)
        return result / self.interval * self.scale_factor


class MLP_norm(nn.Module):
    """(RECALLED-matgl) Linear stack, activation after each layer except the last unless activate_last."""

    def __init__(self, dims, activation=None, activate_last=False, use_bias=True, bias_last=True):
        super().__init__()
        self.layers = nn.ModuleList()
        self._depth = len(dims) - 1
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            bias = use_bias if i < self._depth - 1 else (use_bias and bias_last)
            self.layers.append(nn.Linear(a, b, bias=bias))
        self.activation = activation if activation is not None else nn.SiLU()
        self.activate_last = activate_last

    def forward(self, x):
        for i, lin in enumerate(self.layers):
            x = lin(x)
            if i < self._depth - 1 or self.activate_last:
                x = self.activation(x)
        return x


class GatedMLP_norm(nn.Module):
    """(RECALLED-matgl) layers(z) * sigmoid(gates(z)); `layers` activates its last Linear, `gates` not."""

    def __init__(self, in_feats, dims):
        super().__init__()
        self.layers = MLP_norm([in_feats, *dims], nn.SiLU(), activate_last=True)
        self.gates = MLP_norm([in_feats, *dims], nn.SiLU(), activate_last=False)
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        return self.layers(x) * self.sigmoid(self.gates(x))


class CHGNetGraphConv(nn.Module):
    """(RECALLED-matgl) atom-graph conv; bond update disabled (bond_update_hidden_dims=None)."""

    def __init__(self, dim_atom, dim_bond, hidden):
        super().__init__()
        self.node_update_func = GatedMLP_norm(2 * dim_atom + dim_bond, [*hidden, dim_atom])
        self.node_out_func = nn.Linear(dim_atom, dim_atom, bias=False)
        self.edge_update_func = None
        self.edge_out_func = None
        self.node_weight_func = None
        self.edge_weight_func = None


class CHGNetAtomGraphBlock(nn.Module):
    def __init__(self, dim_atom, dim_bond, hidden):
        super().__init__()
        self.conv_layer = CHGNetGraphConv(dim_atom, dim_bond, hidden)
        self.dropout = nn.Identity()

    def forward(self, src, dst, x, e, w_ab):
        """x' = x + W_out * sum_{e->dst} GatedMLP([x_src | e | x_dst]) * w_ab[e]  (SURVEY §8 a9)."""
        c = self.conv_layer
        z = torch.hstack([x[src], e, x[dst]])
        msg = c.node_update_func(z)
        if w_ab is not None:
            msg = msg * w_ab
        agg = torch.zeros_like(x).index_add_(0, dst, msg)
        return x + c.node_out_func(agg), e


class CHGNetLineGraphConv(nn.Module):
    def __init__(self, dim_atom, dim_bond, dim_angle, node_hidden, edge_hidden):
        super().__init__()
        din = 2 * dim_bond + dim_angle + dim_atom
        self.node_update_func = GatedMLP_norm(din, [*node_hidden, dim_bond])
        self.node_out_func = nn.Linear(dim_bond, dim_bond, bias=False)
        self.edge_update_func = GatedMLP_norm(din, [*edge_hidden, dim_angle]) if edge_hidden is not None else None
        self.node_weight_func = None


class CHGNetBondGraphBlock(nn.Module):
    def __init__(self, dim_atom, dim_bond, dim_angle, node_hidden, edge_hidden):
        super().__init__()
        self.conv_layer = CHGNetLineGraphConv(dim_atom, dim_bond, dim_angle, node_hidden, edge_hidden)
        self.bond_dropout = nn.Identity()
        self.angle_dropout = nn.Identity()

    def node_phase(self, la, lb, center, x, h, ang, w3b):
        """chgnet_layers.py:101-107 + matgl node_update_ (SURVEY §8 a11):
        h_b += (W_out * sum_a GatedMLP([h_a | ang | x_c | h_b])) * w3b[b]."""
        c = self.conv_layer
        z = torch.hstack([h[la], ang, x[center], h[lb]])
        m = c.node_update_func(z)
        agg = torch.zeros_like(h).index_add_(0, lb, m)
        upd = c.node_out_func(agg)
        if w3b is not None:
            upd = upd * w3b
        return h + upd

    def edge_phase(self, la, lb, center, x, h, ang):
        """chgnet_layers.py:109-118 + matgl edge_update_ (SURVEY §8 a12), uses the *new* h."""
        c = self.conv_layer
        if c.edge_update_func is None:
            return ang
        z = torch.hstack([h[la], ang, x[center], h[lb]])
        return ang + c.edge_update_func(z)


class CHGNetRef(nn.Module):
    """Attribute tree mirrors matgl.models.CHGNet (SURVEY §8c)."""

    def __init__(self, element_types=DEFAULT_ELEMENTS, dim=64, cutoff=5.0, threebody_cutoff=3.0,
                 cutoff_exponent=5, max_n=9, max_f=4, num_blocks=4, seed=0):
        super().__init__()
        g = torch.random.get_rng_state()
        torch.manual_seed(seed)
        self.element_types = tuple(element_types)
        self.cutoff = cutoff
        self.three_body_cutoff = threebody_cutoff
        self.cutoff_exponent = cutoff_exponent
        self.n_blocks = num_blocks
        self.max_n = max_n
        self.max_f = max_f
        self.use_bond_graph = True
        self.readout_field = "atom_feat"
        self.readout_operation = "sum"
        self.state_embedding = None
        self.is_intensive = False
        self.bond_expansion = RadialBesselFunction(max_n, cutoff, learnable=True)
        self.threebody_bond_expansion = RadialBesselFunction(max_n, threebody_cutoff, learnable=True)
        self.angle_expansion = FourierExpansion(max_f, learnable=True)
        nfour = 2 * max_f + 1
        self.atom_embedding = nn.Embedding(len(self.element_types), dim)
        self.bond_embedding = MLP_norm([max_n, dim], nn.SiLU(), activate_last=False, bias_last=False)
        self.angle_embedding = MLP_norm([nfour, dim], nn.SiLU(), activate_last=False, bias_last=False)
        self.atom_bond_weights = nn.Linear(max_n, dim, bias=False)
        self.bond_bond_weights = nn.Linear(max_n, dim, bias=False)
        self.threebody_bond_weights = nn.Linear(max_n, dim, bias=False)
        self.atom_graph_layers = nn.ModuleList(
            [CHGNetAtomGraphBlock(dim, dim, (dim,)) for _ in range(num_blocks)])
        self.bond_graph_layers = nn.ModuleList(
            [CHGNetBondGraphBlock(dim, dim, dim, (dim,), ()) for _ in range(num_blocks - 1)])
        self.sitewise_readout = nn.Linear(dim, 1)
        self.final_layer = MLP_norm([dim, dim, dim, 1], nn.SiLU(), activate_last=False)
        torch.random.set_rng_state(g)

    # ------------------------------------------------------------------
    def forward_graph(self, pos, vec, i1, i2, bond_edges, la, lb, center, node_types, taps=None):
        """chgnet.py:100-453 over the global graph. i1 = DGL src (centre), i2 = DGL dst (neighbour);
        messages aggregate at i2 (subgraph_creation_fast.c:166-196 passes index_1 as src_nodes).
        bond_edges[b] = edge id of bond node b; (la -> lb, centre) = line-graph edges."""
        d = torch.linalg.norm(vec, dim=1)
        rbf = self.bond_expansion(d)
        be = polynomial_cutoff(rbf, self.cutoff, self.cutoff_exponent) * rbf  # chgnet.py:116-124
        bvec = vec[bond_edges]
        bd = d[bond_edges]
        rbf3 = self.threebody_bond_expansion(bd)
        tbe = polynomial_cutoff(rbf3, self.three_body_cutoff, self.cutoff_exponent) * rbf3  # :171-182
        # compute_theta with src_bond_sign = -1 (chgnet.py:190-194)
        v1 = -bvec[la]
        v2 = bvec[lb]
        cosv = (v1 * v2).sum(1) / (torch.linalg.norm(v1, dim=1) * torch.linalg.norm(v2, dim=1))
        cosv = cosv.clamp(min=-1 + 1e-7, max=1 - 1e-7)
        theta = torch.acos(cosv)
        fourier = self.angle_expansion(theta)

        x = self.atom_embedding(node_types)
        e = self.bond_embedding(be)
        ang = self.angle_embedding(fourier)
        h = e[bond_edges]  # edge_to_bond (dist.py:671-676)
        w_ab = self.atom_bond_weights(be)
        w_3b = self.threebody_bond_weights(tbe)
        if taps is not None:
            taps.update(d=d, be=be, tbe=tbe, theta=theta, fourier=fourier, x0=x, e0=e, ang0=ang, h0=h,
                        w_ab=w_ab, w_3b=w_3b)
        for l in range(self.n_blocks - 1):
            x, e = self.atom_graph_layers[l](i1, i2, x, e, w_ab)
            h = e[bond_edges]  # dist.py:666-668
            h = self.bond_graph_layers[l].node_phase(la, lb, center, x, h, ang, w_3b)
            e = e.index_copy(0, bond_edges, h)  # bond_to_edge (dist.py:700-702)
            ang = self.bond_graph_layers[l].edge_phase(la, lb, center, x, h, ang)
            if taps is not None:
                taps[f"x{l + 1}"] = x
                taps[f"h{l + 1}"] = h
                taps[f"ang{l + 1}"] = ang
        site = self.sitewise_readout(x)
        x, e = self.atom_graph_layers[-1](i1, i2, x, e, w_ab)
        if taps is not None:
            taps[f"x{self.n_blocks}"] = x
        e_atom = self.final_layer(x)
        if taps is not None:
            taps["e_atom"] = e_atom
        return e_atom.sum(), site


def build_line_graph(i1, i2, bond_mask):
    """Global line graph in the reference's convention (subgraph_creation_utils.c:703-751):
    bond nodes = edges with bond_mask; line edge a=(s->d) -> b=(d->x) iff x != s; centre = d."""
    bond_edges = np.nonzero(bond_mask)[0]
    bs, bd = i1[bond_edges], i2[bond_edges]
    nb = len(bond_edges)
    n = int(max(i1.max(), i2.max())) + 1 if len(i1) else 0
    order = np.argsort(bs, kind="stable")  # out-bonds grouped by src
    start = np.searchsorted(bs[order], np.arange(n), side="left")
    end = np.searchsorted(bs[order], np.arange(n), side="right")
    la, lb, ce = [], [], []
    for a in range(nb):
        d = bd[a]
        s = bs[a]
        for t in range(start[d], end[d]):
            b = order[t]
            if bd[b] == s:
                continue
            la.append(a)
            lb.append(b)
            ce.append(d)
    return (bond_edges, np.array(la, dtype=np.int64), np.array(lb, dtype=np.int64),
            np.array(ce, dtype=np.int64))


def potential_ref(model, atoms, graph=None, calc_forces=True, calc_stresses=True, data_mean=0.0,
                  data_std=1.0, element_refs=None, dtype=torch.float32, taps=None):
    """Restates Potential_Dist.forward (pes.py:50-146) + potential_forward_dist geometry
    (chgnet.py:33-100) for the global graph. Returns (E[1], F[N,3], stress[3,3] GPa, site[N,1])."""
    from oracle.graph_ref import neighbor_list

    lattice_np = np.array(atoms.get_cell())
    cart = np.array(atoms.get_positions(wrap=False))
    pbc = atoms.get_pbc().astype(np.int64)
    if graph is None:
        i1, i2, off, _d2, bond = neighbor_list(cart, lattice_np, pbc, float(model.cutoff),
                                               float(model.three_body_cutoff))
        graph = (i1, i2, off, bond)
    i1, i2, off, bond = graph
    bond_edges, la, lb, ce = build_line_graph(i1, i2, bond)
    model = model.to(dtype)
    lattice = torch.tensor(lattice_np, dtype=dtype)
    strain = torch.zeros(3, 3, dtype=dtype, requires_grad=calc_stresses)
    lattice = lattice @ (torch.eye(3, dtype=dtype) + strain)
    frac = torch.tensor(atoms.get_scaled_positions(False), dtype=dtype)
    pos = frac @ lattice
    if calc_forces:
        pos.retain_grad()
    offshift = torch.tensor(off, dtype=dtype) @ lattice
    t = lambda a: torch.as_tensor(a, dtype=torch.int64)
    vec = pos[t(i2)] + offshift - pos[t(i1)]  # chgnet.py:96-99
    el2idx = {el: k for k, el in enumerate(model.element_types)}
    node_types = t(np.array([el2idx[s] for s in atoms.get_chemical_symbols()]))
    e_raw, site = model.forward_graph(pos, vec, t(i1), t(i2), t(bond_edges), t(la), t(lb), t(ce),
                                      node_types, taps=taps)
    total = data_std * e_raw + data_mean
    if element_refs is not None:
        total = total + torch.as_tensor(np.asarray(element_refs), dtype=dtype)[node_types].sum()
    forces = stress = None
    if calc_forces or calc_stresses:
        total.backward()
        if calc_forces:
            forces = -pos.grad
        if calc_stresses:
            vol = abs(np.linalg.det(lattice_np))
            stress = strain.grad / vol * 160.21766208  # pes.py:140-145
    return total.detach().reshape(1), forces, stress, site.detach()
