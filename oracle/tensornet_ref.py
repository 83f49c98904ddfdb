"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Pure-PyTorch (CPU) restatement of the arithmetic behind the reference's TensorNet path (SURVEY.md §8(f).2):

  control flow / DistMLIP-specific behaviour .... DistMLIP/implementations/matgl/models/tensornet.py:10-161
                                                 DistMLIP/implementations/matgl/pes.py:50-146
  layer internals ............................... matgl @ git 5171392 (pyproject.toml:26-28): `matgl.models.TensorNet`,
                                                 `matgl.layers.TensorEmbedding`, `TensorNetInteraction`, `BondExpansion`,
                                                 `WeightedReadOut`, `matgl.utils.maths.{decompose_tensor, tensor_norm,
                                                 vector_to_skewtensor, vector_to_symtensor}`, `matgl.utils.cutoff.
                                                 cosine_cutoff` -- NOT in the reference repository:
                                                 restated from memory of that code ("RECALLED-matgl"), which itself
                                                 follows the published TensorNet architecture (Simeon & De Fabritiis 2023).

PARITY UNPINNED: the reference ships no tests / golden vectors for the model arithmetic and matgl + dgl are not
available to the tests, so nothing in this file has been checked against a run
of the real reference.

The attribute tree and `state_dict` keys mirror matgl's `TensorNet` as `TensorNet_Dist.enable_distributed_mode`
dereferences it (tensornet.py:163-204: `bond_expansion`, `tensor_embedding`, `layers`, `linear`, `final_layer`,
`out_norm`, `element_types`) so that `TensorNet_Dist.from_existing` accepts either a real matgl model or this one.

One deliberate difference from the reference's multi-partition run is documented in DESIGN.md: the reference does not
exchange the embedded tensors of the halo atoms before the first interaction layer (tensornet.py:104-127: the first
`atom_transfer` follows layer 0), so with more than one partition its first layer reads zero tensors for the halo
sources and the result depends on the partition count.  This oracle is the single-graph evaluation (what plain matgl
computes, and what the reference computes on one partition); the engine exchanges after the embedding to reproduce it
for every partition count.
"""
from __future__ import annotations

import math

import numpy as np
import torch
from torch import nn

from oracle.chgnet_ref import DEFAULT_ELEMENTS


def cosine_cutoff(r, cutoff):
    """matgl.utils.cutoff.cosine_cutoff (RECALLED-matgl)."""
    return torch.where(r <= cutoff, 0.5 * (torch.cos(math.pi * r / cutoff) + 1.0), torch.zeros_like(r))


def vector_to_skewtensor(v):
    """[[0,-z,y],[z,0,-x],[-y,x,0]] (matgl.utils.maths, RECALLED-matgl)."""
    z = torch.zeros_like(v[:, 0])
    t = torch.stack((z, -v[:, 2], v[:, 1], v[:, 2], z, -v[:, 0], -v[:, 1], v[:, 0], z), dim=1)
    return t.view(-1, 3, 3)


def vector_to_symtensor(v):
    """v v^T symmetrised minus mean(diag) * I (matgl.utils.maths, RECALLED-matgl)."""
    t = torch.matmul(v.unsqueeze(-1), v.unsqueeze(-2))
    eye = torch.eye(3, dtype=v.dtype)
    I = t.diagonal(offset=0, dim1=-1, dim2=-2).mean(-1)[..., None, None] * eye
    return 0.5 * (t + t.transpose(-2, -1)) - I


def decompose_tensor(t):
    """(I, A, S): isotropic, antisymmetric, symmetric-traceless parts (matgl.utils.maths, RECALLED-matgl)."""
    eye = torch.eye(3, dtype=t.dtype)
    I = t.diagonal(offset=0, dim1=-1, dim2=-2).mean(-1)[..., None, None] * eye
    A = 0.5 * (t - t.transpose(-2, -1))
    S = 0.5 * (t + t.transpose(-2, -1)) - I
    return I, A, S


def tensor_norm(t):
    return (t**2).sum((-2, -1))


class GaussianExpansion(nn.Module):
    """matgl.layers._basis.GaussianExpansion (RECALLED-matgl): exp(-width (d - mu_k)^2), fixed centres."""

    def __init__(self, initial=0.0, final=4.0, num_centers=20, width=0.5):
        super().__init__()
        self.centers = nn.Parameter(torch.linspace(initial, final, num_centers), requires_grad=False)
        self.width = float(1.0 / torch.diff(self.centers).mean()) if width is None else float(width)

    def forward(self, d):
        return torch.exp(-self.width * (d[:, None] - self.centers[None, :]) ** 2)


class BondExpansion(nn.Module):
    """matgl.layers.BondExpansion with rbf_type="Gaussian" (TensorNet's default; RECALLED-matgl)."""

    def __init__(self, cutoff=5.0, num_centers=32, width=0.5, final=None):
        super().__init__()
        self.rbf_type = "Gaussian"
        self.rbf = GaussianExpansion(0.0, cutoff + 1.0 if final is None else final, num_centers, width)

    def forward(self, d):
        return self.rbf(d)


class TensorEmbedding(nn.Module):
    """matgl.layers._embedding.TensorEmbedding (RECALLED-matgl)."""

    def __init__(self, units, degree_rbf, ntypes_node, cutoff):
        super().__init__()
        self.units, self.cutoff = units, cutoff
        self.distance_proj1 = nn.Linear(degree_rbf, units)
        self.distance_proj2 = nn.Linear(degree_rbf, units)
        self.distance_proj3 = nn.Linear(degree_rbf, units)
        self.emb = nn.Embedding(ntypes_node, units)
        self.emb2 = nn.Linear(2 * units, units)
        self.linears_tensor = nn.ModuleList([nn.Linear(units, units, bias=False) for _ in range(3)])
        self.linears_scalar = nn.ModuleList([nn.Linear(units, 2 * units), nn.Linear(2 * units, 3 * units)])
        self.init_norm = nn.LayerNorm(units)
        self.act = nn.SiLU()

    def forward(self, src, dst, node_type, d, vec, edge_attr, n, taps=None):
        z = self.emb(node_type)
        Zij = self.emb2(torch.cat([z[src], z[dst]], dim=1))[..., None, None]  # [E,units,1,1]
        C = cosine_cutoff(d, self.cutoff).reshape(-1, 1, 1, 1) * Zij
        vn = vec / torch.norm(vec, dim=1).unsqueeze(1)
        eye = torch.eye(3, dtype=vec.dtype)[None, None]
        Iij = self.distance_proj1(edge_attr)[..., None, None] * C * eye
        Aij = self.distance_proj2(edge_attr)[..., None, None] * C * vector_to_skewtensor(vn)[:, None]
        Sij = self.distance_proj3(edge_attr)[..., None, None] * C * vector_to_symtensor(vn)[:, None]
        zero = torch.zeros(n, self.units, 3, 3, dtype=vec.dtype)
        scalars = zero.index_add(0, dst, Iij)  # dgl update_all(copy_e, sum): messages summed at the destination
        skew = zero.index_add(0, dst, Aij)
        traceless = zero.index_add(0, dst, Sij)
        norm = self.init_norm(tensor_norm(scalars + skew + traceless))
        mix = lambda lin, t: lin(t.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
        scalars, skew, traceless = (mix(self.linears_tensor[0], scalars), mix(self.linears_tensor[1], skew),
                                    mix(self.linears_tensor[2], traceless))
        for lin in self.linears_scalar:
            norm = self.act(lin(norm))
        norm = norm.reshape(norm.shape[0], self.units, 3)
        X = (scalars * norm[..., 0, None, None] + skew * norm[..., 1, None, None]
             + traceless * norm[..., 2, None, None])
        return X


class TensorNetInteraction(nn.Module):
    """matgl.layers._graph_convolution.TensorNetInteraction (RECALLED-matgl)."""

    def __init__(self, num_rbf, units, cutoff, equivariance_invariance_group="O(3)"):
        super().__init__()
        self.units, self.cutoff = units, cutoff
        self.equivariance_invariance_group = equivariance_invariance_group
        self.linears_scalar = nn.ModuleList([nn.Linear(num_rbf, units), nn.Linear(units, 2 * units),
                                             nn.Linear(2 * units, 3 * units)])
        self.linears_tensor = nn.ModuleList([nn.Linear(units, units, bias=False) for _ in range(6)])
        self.act = nn.SiLU()

    def forward(self, src, dst, d, edge_attr, X):
        C = cosine_cutoff(d, self.cutoff)
        f = edge_attr
        for lin in self.linears_scalar:
            f = self.act(lin(f))
        f = (f * C.view(-1, 1)).reshape(f.shape[0], self.units, 3)
        X = X / (tensor_norm(X) + 1)[..., None, None]
        I, A, S = decompose_tensor(X)
        mix = lambda lin, t: lin(t.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
        I, A, S = mix(self.linears_tensor[0], I), mix(self.linears_tensor[1], A), mix(self.linears_tensor[2], S)
        Y = I + A + S
        zero = torch.zeros_like(X)
        Im = zero.index_add(0, dst, f[..., 0, None, None] * I[src])  # message = factor * tensor[src], summed at dst
        Am = zero.index_add(0, dst, f[..., 1, None, None] * A[src])
        Sm = zero.index_add(0, dst, f[..., 2, None, None] * S[src])
        msg = Im + Am + Sm
        if self.equivariance_invariance_group == "O(3)":
            I, A, S = decompose_tensor(torch.matmul(msg, Y) + torch.matmul(Y, msg))
        else:  # "SO(3)"
            I, A, S = decompose_tensor(2 * torch.matmul(Y, msg))
        normp1 = (tensor_norm(I + A + S) + 1)[..., None, None]
        I, A, S = I / normp1, A / normp1, S / normp1
        I, A, S = mix(self.linears_tensor[3], I), mix(self.linears_tensor[4], A), mix(self.linears_tensor[5], S)
        dX = I + A + S
        return X + dX + torch.matmul(dX, dX)


class GatedMLP(nn.Module):
    """matgl.layers._core.GatedMLP (RECALLED-matgl): SiLU chain times a sigmoid-terminated gate chain; activations are
    modules of the Sequential, so the Linear layers sit at even indices."""

    def __init__(self, in_feats, dims, activate_last=True):
        super().__init__()
        self.dims = [in_feats, *dims]
        depth = len(dims)
        self.layers, self.gates = nn.Sequential(), nn.Sequential()
        for i, (a, b) in enumerate(zip(self.dims[:-1], self.dims[1:])):
            self.layers.append(nn.Linear(a, b))
            self.gates.append(nn.Linear(a, b))
            if i < depth - 1:
                self.layers.append(nn.SiLU())
                self.gates.append(nn.SiLU())
            else:
                if activate_last:
                    self.layers.append(nn.SiLU())
                self.gates.append(nn.Sigmoid())

    def forward(self, x):
        return self.layers(x) * self.gates(x)


class WeightedReadOut(nn.Module):
    """matgl.layers._readout.WeightedReadOut (RECALLED-matgl): `gated` is what tensornet.py:134 calls."""

    def __init__(self, in_feats, dims, num_targets):
        super().__init__()
        self.dims = [in_feats, *dims, num_targets]
        self.gated = GatedMLP(in_feats=in_feats, dims=self.dims, activate_last=False)


class TensorNetRef(nn.Module):
    """Module tree of matgl `TensorNet` with the constructor defaults (units 64, nblocks 2, num_rbf 32, Gaussian
    expansion of width 0.5 on [0, cutoff + 1], swish, cutoff 5, O(3), is_intensive=False, no state features)."""

    def __init__(self, element_types=DEFAULT_ELEMENTS, units=64, nblocks=2, num_rbf=32, cutoff=5.0, width=0.5,
                 equivariance_invariance_group="O(3)", ntargets=1):
        super().__init__()
        self.element_types = tuple(element_types)
        self.units, self.nblocks, self.num_rbf, self.cutoff = units, nblocks, num_rbf, cutoff
        self.equivariance_invariance_group = equivariance_invariance_group
        self.is_intensive = False
        self.rbf_type = "Gaussian"
        self.activation_type = "swish"
        self.bond_expansion = BondExpansion(cutoff=cutoff, num_centers=num_rbf, width=width)
        self.tensor_embedding = TensorEmbedding(units, num_rbf, len(self.element_types), cutoff)
        self.layers = nn.ModuleList([TensorNetInteraction(num_rbf, units, cutoff, equivariance_invariance_group)
                                     for _ in range(nblocks)])
        self.out_norm = nn.LayerNorm(3 * units)
        self.linear = nn.Linear(3 * units, units)
        self.final_layer = WeightedReadOut(in_feats=units, dims=[units, units], num_targets=ntargets)

    def forward_graph(self, vec, src, dst, node_types, taps=None):
        """tensornet.py:84-147 for one graph. Returns sum of atomic energies (unscaled)."""
        n = node_types.shape[0]
        d = torch.linalg.norm(vec, dim=1)
        edge_attr = self.bond_expansion(d)
        X = self.tensor_embedding(src, dst, node_types, d, vec, edge_attr, n)
        if taps is not None:
            taps["X0"] = X.detach()
        for l, layer in enumerate(self.layers):
            X = layer(src, dst, d, edge_attr, X)
            if taps is not None:
                taps[f"X{l + 1}"] = X.detach()
        I, A, S = decompose_tensor(X)
        x = torch.cat((tensor_norm(I), tensor_norm(A), tensor_norm(S)), dim=-1)
        x = self.linear(self.out_norm(x))
        e_atom = self.final_layer.gated(x)
        if taps is not None:
            taps["e_atom"] = e_atom.detach()
        return torch.squeeze(e_atom.sum(dim=0))


def potential_ref(model, atoms, graph=None, calc_forces=True, calc_stresses=True, data_mean=0.0, data_std=1.0,
                  element_refs=None, dtype=torch.float32, taps=None):
    """Potential_Dist.forward (pes.py:50-146) + TensorNet_Dist.potential_forward_dist geometry (tensornet.py:20-90) on
    the global graph (use_bond_graph False, three_body_cutoff 0: pes.py:79-80). Returns (E[1], F[N,3], stress GPa)."""
    from oracle.graph_ref import neighbor_list

    lattice_np = np.array(atoms.get_cell())
    cart = np.array(atoms.get_positions(wrap=False))
    pbc = atoms.get_pbc().astype(np.int64)
    if graph is None:
        i1, i2, off, _d2, _bond = neighbor_list(cart, lattice_np, pbc, float(model.cutoff), 0.0)
        graph = (i1, i2, off)
    i1, i2, off = graph[:3]
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
    vec = pos[t(i2)] + offshift - pos[t(i1)]  # tensornet.py:84-88
    el2idx = {el: k for k, el in enumerate(model.element_types)}
    node_types = t(np.array([el2idx[s] for s in atoms.get_chemical_symbols()]))
    e_raw = model.forward_graph(vec, t(i1), t(i2), node_types, taps=taps)
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
    return total.detach().reshape(1), forces, stress
