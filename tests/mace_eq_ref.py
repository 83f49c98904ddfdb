"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

CPU restatement (torch, float64) of mace's `ScaleShiftMACE` with equivariant hidden features C x 0e + C x 1o (the shape of
MACE-MP-0 "medium"), with mace's attribute tree and state_dict names.  It extends oracle/mace_ref.py (the scalar model,
whose conventions hold here unchanged and whose building blocks, `potential_ref` and `atomic_virials_ref` are reused)
by the conventions that only a 1o hidden feature needs.  mace and e3nn are not available here, so, as there, every
convention below is recalled, not pinned against a mace checkout:

  * layer shapes: layer 0 takes C x 0e; every layer t < T - 1 gives 0e+1o, the last gives C x 0e (mace's
    hidden_irreps_out = hidden_irreps[0] for the last interaction).  h[t] (0 < t < T) is [n, 4, C]: l = 0, then l = 1
    with m = 0..2 in the `sh_basis` order (x, y, z).  This is also the layout of the `h<t>` taps.
  * linear_up / products.t.linear on 0e+1o: one [C, C] / sqrt(C) block per l, ascending l; the l = 1 block acts on each
    of the 3 components.
  * conv_tp ("uvu", mace's tp_out_irreps_with_instructions; `conv_paths`): the paths (l_in, l_sh) -> l_out with
    |l_in - l_sh| <= l_out <= l_in + l_sh, l_out <= max_ell and parity p_in (-1)^l_sh = (-1)^l_out, stable-sorted by l_out
    (10 paths for max_ell 3, 7 for 2, 4 for 1).  Path p adds R[e][p][c] sqrt(2 l_out + 1) sum CG[m1, m2, m3]
    u[src][c][l_in m1] Y[e][l_sh m2] to component (l_out, m3); CG = `make_cg` (e3nn wigner_3j with "component" irrep and
    "element" path normalisation).  For (0, l) -> l this is the scalar model's path constant 1.  The radial MLP ends in
    n_paths * C outputs, path-major.
  * interactions.t.linear from the per-path blocks: flat [C, C] per path in path order; output l divided by
    sqrt(n_paths(l) * C) and by avg_num_neighbors.
  * skip_tp of a residual block with 0e+1o input: paths (0e, elem) -> 0e and, when the layer gives 1o, (1o, elem) -> 1o,
    [C, n_elem, C] / sqrt(C n_elem) each, ascending l.  A non-residual block keeps the skip on the target irreps.  A
    residual layer 0 (0e input) giving 0e+1o has the 0e path only.
  * symmetric contraction: contractions.0 gives 0e (as in the scalar model); contractions.1 gives 1o from U_matrix_nu
    [3, nsh, ..., K] (`make_u_vec`, output component first) and its own weights_max / weights.{j} [n_elem, K, C]:
    B1[c, m] = sum_nu sum_k w_nu[z, k, c] sum U_nu[m, i1..inu, k] A[c, i1] ... A[c, inu].
  * a LinearReadoutBlock on 0e+1o reads the 0e block only (weight [C]).

The random U bases (`make_u`, `make_u_vec`) are null-space bases of degenerate spaces: LAPACK may return another
orthonormal basis of the same space under other threading, so compare the engine with the oracle on one model object.
"""
from __future__ import annotations

import functools
import itertools
import math

import numpy as np
import torch
from torch import nn

from oracle import mace_ref as _s
from oracle.mace_ref import (FullyConnectedNet, _random_rotation, _W, atomic_virials_ref, l_of_index, nsh_of,  # noqa: F401
                             potential_ref, species_index, wigner_d)


# ------------------------------------------------------------------------------------------ coupling and U tensors
@functools.lru_cache(maxsize=None)
def make_cg(l1, l2, l3, seed=0):
    """Real coupling tensor [2 l1 + 1, 2 l2 + 1, 2 l3 + 1] in the basis of `sh_basis`: the null space of
    D_l1 (x) D_l2 (x) D_l3 - I under two random rotations and the inversion, unit Frobenius norm.  Sign rule: the first
    entry (C order) with |x| > 1e-6 is positive.  Raises ValueError when no such tensor exists."""
    rng = np.random.default_rng(seed)
    ls = (l1, l2, l3)
    blk = lambda D, l: D[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2]  # noqa: E731
    gens = []
    for _ in range(2):
        D = wigner_d(_random_rotation(rng), 3, rng)
        gens.append([blk(D, l) for l in ls])
    gens.append([(-1.0) ** l * torch.eye(2 * l + 1, dtype=torch.float64) for l in ls])
    dim = (2 * l1 + 1) * (2 * l2 + 1) * (2 * l3 + 1)
    M = torch.cat([torch.kron(torch.kron(a, b), c) - torch.eye(dim, dtype=torch.float64) for a, b, c in gens], dim=0)
    _, sv, Vh = torch.linalg.svd(M)
    null = Vh[sv < 1e-9]
    if null.shape[0] != 1:
        raise ValueError(f"no coupling {ls} (null space of dimension {null.shape[0]})")
    cg = null[0] / torch.linalg.norm(null[0])
    first = cg[cg.abs() > 1e-6][0]
    return (cg * torch.sign(first)).reshape(2 * l1 + 1, 2 * l2 + 1, 2 * l3 + 1).contiguous()


def conv_paths(max_ell, hidden_l=0):
    """(l_in, l_sh, l_out) of conv_tp for node features 0e (+ 1o when hidden_l = 1), in mace's order: enumerated over
    l_in, l_sh, l_out, kept when l_out <= max_ell and the parities match, then stable-sorted by l_out"""
    paths = []
    for l_in in range(hidden_l + 1):
        for l_sh in range(max_ell + 1):
            for l_out in range(abs(l_in - l_sh), min(l_in + l_sh, max_ell) + 1):
                if (l_in + l_sh + l_out) % 2 == 0:  # p_in (-1)^l_sh = (-1)^l_out with p_in = (-1)^l_in (0e, 1o)
                    paths.append((l_in, l_sh, l_out))
    return sorted(paths, key=lambda p: p[2])


@functools.lru_cache(maxsize=None)
def make_u_vec(max_ell, nu, seed=0):
    """oracle/mace_ref.py `make_u` with a leading 1o output axis: an orthonormal basis of the tensors [3] + [nsh]*nu,
    symmetric in the nu input indices, with D_1(g) (x) D(g)^{(x)nu} T = T for two random rotations and the inversion
    (-1 on the output axis).  One l-tuple of the input indices per basis tensor, so U stays sparse.
    Returns [3] + [nsh]*nu + [K] float64."""
    rng = np.random.default_rng(seed)
    n = nsh_of(max_ell)
    gens = [wigner_d(_random_rotation(rng), max_ell, rng) for _ in range(2)]
    gens.append(torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64)))
    outs = [D[1:4, 1:4] for D in gens]  # the l = 1 block; -I for the inversion
    lidx = l_of_index(max_ell)
    by_l = {}
    for ms in itertools.combinations_with_replacement(range(n), nu):
        by_l.setdefault(tuple(lidx[i] for i in ms), []).append(ms)
    out = []
    for key in sorted(by_l):
        multisets = by_l[key]
        nm = len(multisets)
        S = torch.zeros(3 * nm, 3, *([n] * nu), dtype=torch.float64)
        for a in range(3):
            for m, ms in enumerate(multisets):
                for perm in set(itertools.permutations(ms)):
                    S[(a * nm + m, a) + perm] = 1.0
        S = S / torch.linalg.norm(S.reshape(3 * nm, -1), dim=1).reshape(-1, *([1] * (nu + 1)))
        blocks = []
        for Do, D in zip(outs, gens):
            T = torch.movedim(torch.tensordot(S, Do, dims=([1], [1])), -1, 1)
            for ax in range(nu):
                T = torch.movedim(torch.tensordot(T, D, dims=([2 + ax], [1])), -1, 2 + ax)
            blocks.append((T - S).reshape(3 * nm, -1))
        Uv, sv, _ = torch.linalg.svd(torch.cat(blocks, dim=1), full_matrices=False)
        sv_full = torch.zeros(3 * nm, dtype=torch.float64)
        sv_full[: len(sv)] = sv
        null = Uv[:, sv_full < 1e-9]
        out.append(torch.tensordot(null, S, dims=([0], [0])))  # [K_block, 3, n, ..., n]
    return torch.movedim(torch.cat(out, dim=0), 0, -1).contiguous()


# ------------------------------------------------------------------------------------------ modules
class _InteractionEq(nn.Module):
    """interaction with 0e+1o input (layers t >= 1): conv_tp over `conv_paths`, the per-path linear, the skip"""

    def __init__(self, C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors, residual, L_out):
        super().__init__()
        self.C, self.n_elem, self.max_ell, self.residual, self.L_out = C, n_elem, max_ell, residual, L_out
        self.avg_num_neighbors = float(avg_num_neighbors)
        self.hidden_irreps = f"{C}x0e+{C}x1o"  # mace's InteractionBlock attributes (str() of e3nn Irreps)
        self.node_feats_irreps = f"{C}x0e+{C}x1o"
        self.paths = conv_paths(max_ell, 1)
        NP = len(self.paths)
        self.linear_up = _W(2 * C * C)
        self.conv_tp_weights = FullyConnectedNet([num_bessel] + list(radial_mlp) + [NP * C])
        self.linear = _W(NP * C * C)
        self.skip_tp = _W(((1 + L_out) if residual else max_ell + 1) * C * n_elem * C)

    def forward(self, h, z, Y, ef, src, dst):  # h [n, 4, C]
        C, n, L1 = self.C, h.shape[0], self.max_ell + 1
        NP = len(self.paths)
        Wu = self.linear_up.weight.view(2, C, C) / math.sqrt(C)
        u = torch.cat([(h[:, 0] @ Wu[0])[:, None], h[:, 1:] @ Wu[1]], dim=1)[src]  # [E, 4, C]
        R = self.conv_tp_weights(ef).view(-1, NP, C)
        Wlin = self.linear.weight.view(NP, C, C)
        blocks = []
        for lo in range(L1):
            ps = [p for p, pth in enumerate(self.paths) if pth[2] == lo]
            acc = 0.0
            for p in ps:
                li, ls, _ = self.paths[p]
                cg = make_cg(li, ls, lo) * math.sqrt(2 * lo + 1)
                m = torch.einsum("eic,ej,ijk->ekc", u[:, li * li:(li + 1) ** 2], Y[:, ls * ls:(ls + 1) ** 2], cg)
                M = torch.zeros(n, 2 * lo + 1, C, dtype=h.dtype).index_add(0, dst, m * R[:, p, None, :])
                acc = acc + M @ Wlin[p]
            blocks.append(acc / (self.avg_num_neighbors * math.sqrt(len(ps) * C)))
        A = torch.cat(blocks, dim=1)  # [n, nsh, C]
        norm = math.sqrt(C * self.n_elem)
        if self.residual:
            Ws = self.skip_tp.weight.view(1 + self.L_out, C, self.n_elem, C).permute(0, 2, 1, 3)  # [Lw, n_elem, C, C]
            sc = torch.einsum("nc,ncd->nd", h[:, 0], Ws[0][z]) / norm
            if self.L_out:
                sc = torch.cat([sc[:, None], torch.einsum("nmc,ncd->nmd", h[:, 1:], Ws[1][z]) / norm], dim=1)
            return A, sc
        lsel = torch.tensor(l_of_index(self.max_ell))
        Ws = self.skip_tp.weight.view(L1, C, self.n_elem, C)[lsel]
        A = torch.einsum("nic,nicd->nid", A, Ws.permute(2, 0, 1, 3)[z]) / norm
        return A, None


# mace's class names: the engine's wrapper recognises the interaction classes by name
class RealAgnosticResidualInteractionBlock(_InteractionEq):
    def __init__(self, *a, **kw):
        super().__init__(*a, residual=True, **kw)


class RealAgnosticInteractionBlock(_InteractionEq):
    def __init__(self, *a, **kw):
        super().__init__(*a, residual=False, **kw)


class ContractionVec(_s.Contraction):
    """contractions.1: the 1o output, B1 [n, 3, C]"""

    def __init__(self, max_ell, correlation, n_elem, C):
        nn.Module.__init__(self)
        self.correlation = correlation
        for nu in range(1, correlation + 1):
            self.register_buffer(f"U_matrix_{nu}", make_u_vec(max_ell, nu).clone())
        K = lambda nu: getattr(self, f"U_matrix_{nu}").shape[-1]  # noqa: E731
        self.weights_max = nn.Parameter(torch.randn(n_elem, K(correlation), C, dtype=torch.float64) / K(correlation))
        self.weights = nn.ParameterList(
            [nn.Parameter(torch.randn(n_elem, K(nu), C, dtype=torch.float64) / K(nu)) for nu in range(correlation - 1, 0, -1)])

    def forward(self, A, z):
        n, C = A.shape[0], A.shape[2]
        B = torch.zeros(n, 3, C, dtype=A.dtype)
        for nu in range(1, self.correlation + 1):
            U = getattr(self, f"U_matrix_{nu}")
            K = U.shape[-1]
            nz = U.nonzero(as_tuple=True)  # (m, i1..inu, k)
            prod = U[nz][None, :, None] * A[:, nz[1], :]
            for j in range(2, nu + 1):
                prod = prod * A[:, nz[j], :]
            P = torch.zeros(n, 3 * K, C, dtype=A.dtype).index_add(1, nz[0] * K + nz[nu + 1], prod).view(n, 3, K, C)
            B = B + (self.weight_of(nu)[z][:, None] * P).sum(dim=2)
        return B


class SymmetricContractionEq(nn.Module):
    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.contractions = nn.ModuleList([_s.Contraction(max_ell, correlation, n_elem, C),
                                           ContractionVec(max_ell, correlation, n_elem, C)])

    def forward(self, A, z):
        return self.contractions[0](A, z), self.contractions[1](A, z)


class EquivariantProductBasisBlockEq(nn.Module):
    """product block giving 0e+1o: h [n, 4, C]; a scalar skip (0e input) adds to the 0e block only"""

    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.symmetric_contractions = SymmetricContractionEq(max_ell, correlation, n_elem, C)
        self.linear = _W(2 * C * C)
        self.C = C

    def forward(self, A, sc, z):
        B0, B1 = self.symmetric_contractions(A, z)
        W = self.linear.weight.view(2, self.C, self.C) / math.sqrt(self.C)
        h0, h1 = B0 @ W[0], B1 @ W[1]
        if sc is not None:
            h0 = h0 + (sc[:, 0] if sc.dim() == 3 else sc)
            h1 = h1 + sc[:, 1:] if sc.dim() == 3 else h1
        return torch.cat([h0[:, None], h1], dim=1)


class LinearReadoutBlock(_s.LinearReadoutBlock):
    """on 0e+1o features: the 0e block only"""

    def forward(self, h):
        return super().forward(h[:, 0] if h.dim() == 3 else h)


class ScaleShiftMACE(nn.Module):
    """mace.modules.ScaleShiftMACE with hidden_irreps = C x 0e + C x 1o."""

    def __init__(self, atomic_numbers, C=32, max_ell=3, correlation=3, num_interactions=2, r_max=5.0, num_bessel=8,
                 num_polynomial_cutoff=5, radial_mlp=(64, 64, 64), avg_num_neighbors=20.0, mlp_hidden=16,
                 interaction_classes=None, scale=1.0, shift=0.0, atomic_energies=None):
        super().__init__()
        if max_ell < 1:
            raise ValueError("0e+1o hidden features need max_ell >= 1")
        n_elem, T = len(atomic_numbers), num_interactions
        self.register_buffer("atomic_numbers", torch.as_tensor(atomic_numbers, dtype=torch.int64))
        self.register_buffer("r_max", torch.tensor(float(r_max), dtype=torch.float64))
        self.register_buffer("num_interactions", torch.tensor(int(T), dtype=torch.int64))
        self.heads = ["default"]
        self.max_ell, self.correlation = max_ell, correlation
        self.node_embedding = _s.LinearNodeEmbeddingBlock(n_elem, C)
        self.radial_embedding = _s.RadialEmbeddingBlock(r_max, num_bessel, num_polynomial_cutoff)
        if interaction_classes is None:
            interaction_classes = [RealAgnosticInteractionBlock] + [RealAgnosticResidualInteractionBlock] * (T - 1)
        # classes of this module or of oracle/mace_ref.py, told apart by name; layer 0 (0e input) is the scalar model's
        residual = ["Residual" in cls.__name__ for cls in interaction_classes]
        inters = []
        for t in range(T):
            a = (C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors)
            if t == 0:
                it = (_s.RealAgnosticResidualInteractionBlock if residual[0] else _s.RealAgnosticInteractionBlock)(*a)
                it.hidden_irreps, it.node_feats_irreps = f"{C}x0e+{C}x1o", f"{C}x0e"
            else:
                cls = RealAgnosticResidualInteractionBlock if residual[t] else RealAgnosticInteractionBlock
                it = cls(*a, L_out=int(t < T - 1))
            inters.append(it)
        self.interactions = nn.ModuleList(inters)
        self.products = nn.ModuleList(
            [EquivariantProductBasisBlockEq(max_ell, correlation, n_elem, C) if t < T - 1
             else _s.EquivariantProductBasisBlock(max_ell, correlation, n_elem, C) for t in range(T)])
        self.readouts = nn.ModuleList(
            [LinearReadoutBlock(C) for _ in range(T - 1)] + [_s.NonLinearReadoutBlock(C, mlp_hidden)])
        self.scale_shift = _s.ScaleShiftBlock(scale, shift)
        e0 = np.zeros(n_elem) if atomic_energies is None else atomic_energies
        self.atomic_energies_fn = _s.AtomicEnergiesBlock(e0)

    def node_energies(self, vec, src, dst, z, taps=None):
        """(eps_i [n], interaction part e_i [n]); taps: A<t> [n, nsh, C], h<t> [n, 4, C] for 0 < t < T, h<T> [n, C]"""
        d = torch.linalg.norm(vec, dim=1, keepdim=True)
        Y = _s.sh_basis(vec, self.max_ell)
        ef = self.radial_embedding(d)
        h = self.node_embedding(z)
        e = torch.zeros(z.shape[0], dtype=vec.dtype)
        for t, (inter, prod, ro) in enumerate(zip(self.interactions, self.products, self.readouts)):
            A, sc = inter(h, z, Y, ef, src, dst)
            h = prod(A, sc, z)
            e = e + ro(h)
            if taps is not None:
                taps[f"A{t}"], taps[f"h{t + 1}"] = A.detach(), h.detach()
        inter_e = self.scale_shift.scale * e + self.scale_shift.shift
        return self.atomic_energies_fn.atomic_energies[z] + inter_e, inter_e


def make_mace_eq(seed=0, atomic_numbers=(14, 6, 8), **kw):
    """seeded random ScaleShiftMACE with hidden features C x 0e + C x 1o (weights N(0, 1), as e3nn initialises them)"""
    torch.manual_seed(seed)
    kw.setdefault("atomic_energies", np.linspace(-3.0, -1.0, len(atomic_numbers)))
    kw.setdefault("scale", 1.3)
    kw.setdefault("shift", -0.2)
    return ScaleShiftMACE(list(atomic_numbers), **kw)
