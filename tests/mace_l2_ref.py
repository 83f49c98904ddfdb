"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

CPU restatement (torch, float64) of mace's `ScaleShiftMACE` with hidden features C x 0e + C x 1o + C x 2e (the shape of
MACE-MP-0 "large"), with mace's attribute tree and state_dict names.  It extends tests/mace_eq_ref.py (0e+1o), whose
conventions hold here unchanged and whose blocks (`make_cg`, `conv_paths`, `make_u_vec`, the 1o contraction, the linear
readout) are reused, by the conventions that only a 2e hidden feature needs.  As there, every convention below is
recalled, not pinned against a mace checkout:

  * layer shapes: layer 0 takes C x 0e; every layer t < T - 1 gives 0e+1o+2e, the last gives C x 0e.  h[t] (0 < t < T)
    is [n, 9, C]: 0e, then 1o with m = 0..2, then 2e with m = 0..4, in the `sh_basis` order.  This is also the layout of
    the `h<t>` taps.
  * linear_up / products.t.linear on 0e+1o+2e: one [C, C] / sqrt(C) block per l, ascending l; the 2e block acts on each
    of the 5 components.
  * conv_tp uses `conv_paths(max_ell, 2)`: the same parity rule (2e has parity +1 = (-1)^2) and the same stable sort by
    l_out, 11 paths for max_ell 2 and 17 for 3.  Couplings of a path (2, l_sh, l_out) come from `make_cg(2, l_sh, l_out)`.
  * skip_tp of a residual block gains (2e, elem) -> 2e when the layer both takes and gives 2e: three [C, n_elem, C]
    blocks, ascending l.
  * symmetric contraction: contractions.2 gives 2e from U_matrix_nu [5, nsh, ..., K] (`make_u_out(max_ell, nu, 2)`,
    output component first) and its own weights_max / weights.{j} [n_elem, K, C], as contractions.1 gives 1o.

A 2e input needs max_ell >= 2: the 2e output of conv_tp (and of the product) must exist.
"""
from __future__ import annotations

import functools
import itertools
import math

import numpy as np
import torch
from torch import nn

from oracle import mace_ref as _s
from oracle.mace_ref import _random_rotation, _W, l_of_index, nsh_of, wigner_d
from tests import mace_eq_ref as _eq
from tests import mace_zbl_ref as _zbl
from tests.mace_zbl_ref import _CoreRepulsion
from tests.mace_eq_ref import (FullyConnectedNet, LinearReadoutBlock, atomic_virials_ref, conv_paths, make_cg,  # noqa: F401
                               make_u_vec, potential_ref)

HIDDEN_L = 2


@functools.lru_cache(maxsize=None)
def make_u_out(max_ell, nu, l_out, seed=0):
    """`make_u_vec` for an output of degree l_out and parity (-1)^l_out: an orthonormal basis of the tensors
    [2 l_out + 1] + [nsh]*nu, symmetric in the nu input indices, with D_lout(g) (x) D(g)^{(x)nu} T = T for two random
    rotations and the inversion.  l_out = 1 is `make_u_vec` itself (unchanged).  Returns [2 l_out + 1] + [nsh]*nu + [K]."""
    if l_out == 1:  # called as the 0e+1o models call it, so that both share the cached basis
        return make_u_vec(max_ell, nu) if seed == 0 else make_u_vec(max_ell, nu, seed)
    if l_out > max_ell:
        raise ValueError(f"an l = {l_out} output needs max_ell >= {l_out}")
    rng = np.random.default_rng(seed)
    n, no = nsh_of(max_ell), 2 * l_out + 1
    gens = [wigner_d(_random_rotation(rng), max_ell, rng) for _ in range(2)]
    gens.append(torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64)))
    outs = [D[l_out * l_out:(l_out + 1) ** 2, l_out * l_out:(l_out + 1) ** 2] for D in gens]
    lidx = l_of_index(max_ell)
    by_l = {}
    for ms in itertools.combinations_with_replacement(range(n), nu):
        by_l.setdefault(tuple(lidx[i] for i in ms), []).append(ms)
    out = []
    for key in sorted(by_l):
        multisets = by_l[key]
        nm = len(multisets)
        S = torch.zeros(no * nm, no, *([n] * nu), dtype=torch.float64)
        for a in range(no):
            for m, ms in enumerate(multisets):
                for perm in set(itertools.permutations(ms)):
                    S[(a * nm + m, a) + perm] = 1.0
        S = S / torch.linalg.norm(S.reshape(no * nm, -1), dim=1).reshape(-1, *([1] * (nu + 1)))
        blocks = []
        for Do, D in zip(outs, gens):
            T = torch.movedim(torch.tensordot(S, Do, dims=([1], [1])), -1, 1)
            for ax in range(nu):
                T = torch.movedim(torch.tensordot(T, D, dims=([2 + ax], [1])), -1, 2 + ax)
            blocks.append((T - S).reshape(no * nm, -1))
        Uv, sv, _ = torch.linalg.svd(torch.cat(blocks, dim=1), full_matrices=False)
        sv_full = torch.zeros(no * nm, dtype=torch.float64)
        sv_full[: len(sv)] = sv
        null = Uv[:, sv_full < 1e-9]
        out.append(torch.tensordot(null, S, dims=([0], [0])))
    return torch.movedim(torch.cat(out, dim=0), 0, -1).contiguous()


# ------------------------------------------------------------------------------------------ modules
class _InteractionL2(nn.Module):
    """interaction with 0e+1o+2e input (layers t >= 1): conv_tp over `conv_paths(max_ell, 2)`, the per-path linear, the
    skip.  L_out: 2 when the layer gives 0e+1o+2e, 0 for the last layer."""

    def __init__(self, C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors, residual, L_out):
        super().__init__()
        if max_ell < 2:
            raise ValueError("0e+1o+2e hidden features need max_ell >= 2")
        self.C, self.n_elem, self.max_ell, self.residual, self.L_out = C, n_elem, max_ell, residual, L_out
        self.avg_num_neighbors = float(avg_num_neighbors)
        self.hidden_irreps = f"{C}x0e+{C}x1o+{C}x2e"
        self.node_feats_irreps = f"{C}x0e+{C}x1o+{C}x2e"
        self.paths = conv_paths(max_ell, HIDDEN_L)
        NP = len(self.paths)
        self.linear_up = _W((HIDDEN_L + 1) * C * C)
        self.conv_tp_weights = FullyConnectedNet([num_bessel] + list(radial_mlp) + [NP * C])
        self.linear = _W(NP * C * C)
        self.skip_tp = _W(((1 + L_out) if residual else max_ell + 1) * C * n_elem * C)

    def forward(self, h, z, Y, ef, src, dst):  # h [n, 9, C]
        C, n, L1 = self.C, h.shape[0], self.max_ell + 1
        NP = len(self.paths)
        Wu = self.linear_up.weight.view(HIDDEN_L + 1, C, C) / math.sqrt(C)
        u = torch.cat([h[:, l * l:(l + 1) ** 2] @ Wu[l] for l in range(HIDDEN_L + 1)], dim=1)[src]  # [E, 9, C]
        R = self.conv_tp_weights(ef).view(-1, NP, C)
        Wlin = self.linear.weight.view(NP, C, C)
        blocks = []
        for lo in range(L1):
            ps = [p for p, pth in enumerate(self.paths) if pth[2] == lo]
            acc = 0.0
            for p in ps:
                li, ls, _ = self.paths[p]
                cg = make_cg(li, ls, lo) * math.sqrt(2 * lo + 1)
                yc = torch.einsum("ej,ijk->eik", Y[:, ls * ls:(ls + 1) ** 2], cg)  # Y and CG first: no [E, i, j, C]
                m = torch.einsum("eic,eik->ekc", u[:, li * li:(li + 1) ** 2], yc)
                M = torch.zeros(n, 2 * lo + 1, C, dtype=h.dtype).index_add(0, dst, m * R[:, p, None, :])
                acc = acc + M @ Wlin[p]
            blocks.append(acc / (self.avg_num_neighbors * math.sqrt(len(ps) * C)))
        A = torch.cat(blocks, dim=1)  # [n, nsh, C]
        norm = math.sqrt(C * self.n_elem)
        if self.residual:
            Ws = self.skip_tp.weight.view(1 + self.L_out, C, self.n_elem, C).permute(0, 2, 1, 3)  # [Lw, n_elem, C, C]
            if not self.L_out:
                return A, torch.einsum("nc,ncd->nd", h[:, 0], Ws[0][z]) / norm
            sc = [torch.einsum("nmc,ncd->nmd", h[:, l * l:(l + 1) ** 2], Ws[l][z]) / norm for l in range(HIDDEN_L + 1)]
            return A, torch.cat(sc, dim=1)
        lsel = torch.tensor(l_of_index(self.max_ell))
        Ws = self.skip_tp.weight.view(L1, C, self.n_elem, C)[lsel]
        A = torch.einsum("nic,nicd->nid", A, Ws.permute(2, 0, 1, 3)[z]) / norm
        return A, None


class RealAgnosticResidualInteractionBlock(_InteractionL2):
    def __init__(self, *a, **kw):
        super().__init__(*a, residual=True, **kw)


class RealAgnosticInteractionBlock(_InteractionL2):
    def __init__(self, *a, **kw):
        super().__init__(*a, residual=False, **kw)


class ContractionOut(_s.Contraction):
    """contractions.l (l = 1, 2): the output of degree l, B_l [n, 2 l + 1, C]"""

    def __init__(self, max_ell, correlation, n_elem, C, l_out):
        nn.Module.__init__(self)
        self.correlation = correlation
        for nu in range(1, correlation + 1):
            self.register_buffer(f"U_matrix_{nu}", make_u_out(max_ell, nu, l_out).clone())
        K = lambda nu: getattr(self, f"U_matrix_{nu}").shape[-1]  # noqa: E731
        self.weights_max = nn.Parameter(torch.randn(n_elem, K(correlation), C, dtype=torch.float64) / K(correlation))
        self.weights = nn.ParameterList(
            [nn.Parameter(torch.randn(n_elem, K(nu), C, dtype=torch.float64) / K(nu)) for nu in range(correlation - 1, 0, -1)])

    def forward(self, A, z):
        """per element e: U contracted with w_nu[e] first ([no, nsh, .., C]), then with A once per input index, so no
        [n, nonzeros of U, C] product is formed (the 4 096-atom cells of the GPU tests stay within host memory)"""
        n, C = A.shape[0], A.shape[2]
        no = self.U_matrix_1.shape[0]
        B = torch.zeros(n, no, C, dtype=A.dtype)
        for nu in range(1, self.correlation + 1):
            U, W = getattr(self, f"U_matrix_{nu}"), self.weight_of(nu)
            for e in torch.unique(z).tolist():
                sel = (z == e).nonzero(as_tuple=True)[0]
                Ae = A[sel]
                T = torch.einsum("o...ic,nic->no...c", torch.einsum("...k,kc->...c", U, W[e]), Ae)
                for _ in range(nu - 1):
                    T = torch.einsum("no...ic,nic->no...c", T, Ae)
                B = B.index_add(0, sel, T)
        return B


class SymmetricContractionL2(nn.Module):
    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.contractions = nn.ModuleList([_s.Contraction(max_ell, correlation, n_elem, C)] +
                                          [ContractionOut(max_ell, correlation, n_elem, C, l) for l in (1, 2)])

    def forward(self, A, z):
        return [c(A, z) for c in self.contractions]


class EquivariantProductBasisBlockL2(nn.Module):
    """product block giving 0e+1o+2e: h [n, 9, C]; a scalar skip (0e input) adds to the 0e block only"""

    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.symmetric_contractions = SymmetricContractionL2(max_ell, correlation, n_elem, C)
        self.linear = _W((HIDDEN_L + 1) * C * C)
        self.C = C

    def forward(self, A, sc, z):
        B0, B1, B2 = self.symmetric_contractions(A, z)
        W = self.linear.weight.view(HIDDEN_L + 1, self.C, self.C) / math.sqrt(self.C)
        h = torch.cat([(B0 @ W[0])[:, None], B1 @ W[1], B2 @ W[2]], dim=1)
        if sc is None:
            return h
        if sc.dim() == 2:
            return torch.cat([h[:, :1] + sc[:, None], h[:, 1:]], dim=1)
        return h + sc


class ScaleShiftMACE(_eq.ScaleShiftMACE):
    """mace.modules.ScaleShiftMACE with hidden_irreps = C x 0e + C x 1o + C x 2e (node_energies and the taps as in
    tests/mace_eq_ref.py, with h<t> [n, 9, C] for 0 < t < T)."""

    def __init__(self, atomic_numbers, C=32, max_ell=3, correlation=3, num_interactions=2, r_max=5.0, num_bessel=8,
                 num_polynomial_cutoff=5, radial_mlp=(64, 64, 64), avg_num_neighbors=20.0, mlp_hidden=16,
                 interaction_classes=None, scale=1.0, shift=0.0, atomic_energies=None):
        nn.Module.__init__(self)
        if max_ell < 2:
            raise ValueError("0e+1o+2e hidden features need max_ell >= 2")
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
        residual = ["Residual" in cls.__name__ for cls in interaction_classes]
        inters = []
        for t in range(T):
            a = (C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors)
            if t == 0:
                it = (_s.RealAgnosticResidualInteractionBlock if residual[0] else _s.RealAgnosticInteractionBlock)(*a)
                it.hidden_irreps, it.node_feats_irreps = f"{C}x0e+{C}x1o+{C}x2e", f"{C}x0e"
            else:
                cls = RealAgnosticResidualInteractionBlock if residual[t] else RealAgnosticInteractionBlock
                it = cls(*a, L_out=HIDDEN_L if t < T - 1 else 0)
            inters.append(it)
        self.interactions = nn.ModuleList(inters)
        self.products = nn.ModuleList(
            [EquivariantProductBasisBlockL2(max_ell, correlation, n_elem, C) if t < T - 1
             else _s.EquivariantProductBasisBlock(max_ell, correlation, n_elem, C) for t in range(T)])
        self.readouts = nn.ModuleList(
            [LinearReadoutBlock(C) for _ in range(T - 1)] + [_s.NonLinearReadoutBlock(C, mlp_hidden)])
        self.scale_shift = _s.ScaleShiftBlock(scale, shift)
        e0 = np.zeros(n_elem) if atomic_energies is None else atomic_energies
        self.atomic_energies_fn = _s.AtomicEnergiesBlock(e0)


def make_mace_l2(seed=0, atomic_numbers=(14, 6, 8), **kw):
    """seeded random ScaleShiftMACE with hidden features C x 0e + C x 1o + C x 2e (weights N(0, 1))"""
    torch.manual_seed(seed)
    kw.setdefault("atomic_energies", np.linspace(-3.0, -1.0, len(atomic_numbers)))
    kw.setdefault("scale", 1.3)
    kw.setdefault("shift", -0.2)
    return ScaleShiftMACE(list(atomic_numbers), **kw)


def embed_medium(large, medium):
    """Load a 0e+1o model (tests/mace_eq_ref.py, same shapes otherwise) into a 0e+1o+2e one so that both compute the
    same energy: the 2e outputs of every product linear and residual skip are zeroed (h's 2e block stays 0, so no path
    with l_in = 2 contributes), the shared conv_tp paths are moved to their places in `conv_paths(max_ell, 2)`, and each
    path block of interactions.t.linear is scaled by sqrt(np_2(l_out) / np_1(l_out)) against the larger normalisation.
    Returns `large`."""
    sd, md = large.state_dict(), medium.state_dict()
    max_ell = large.max_ell
    with torch.no_grad():
        for k, v in sd.items():
            if k in md and md[k].shape == v.shape:
                v.copy_(md[k])
        T = len(large.interactions)
        C = int(sd["node_embedding.linear.weight"].numel()) // len(large.atomic_numbers)
        p1, p2 = conv_paths(max_ell, 1), conv_paths(max_ell, 2)
        np1 = [sum(p[2] == l for p in p1) for l in range(max_ell + 1)]
        np2 = [sum(p[2] == l for p in p2) for l in range(max_ell + 1)]
        for t in range(1, T):
            pre = f"interactions.{t}."
            up = sd[pre + "linear_up.weight"].view(3, C * C)
            up[:2] = md[pre + "linear_up.weight"].view(2, C * C)
            last = max((k for k in sd if k.startswith(pre + "conv_tp_weights.layer")), key=lambda k: int(k.split(".")[3][5:]))
            Wr, Wr1 = sd[last].view(sd[last].shape[0], len(p2), C), md[last].view(md[last].shape[0], len(p1), C)
            lin, lin1 = sd[pre + "linear.weight"].view(len(p2), C * C), md[pre + "linear.weight"].view(len(p1), C * C)
            for j, p in enumerate(p2):
                if p in p1:
                    i = p1.index(p)
                    Wr[:, j] = Wr1[:, i]
                    lin[j] = lin1[i] * math.sqrt(np2[p[2]] / np1[p[2]])
            sk = sd[pre + "skip_tp.weight"]
            if large.interactions[t].residual and large.interactions[t].L_out:
                sk.view(3, -1)[:2] = md[pre + "skip_tp.weight"].view(2, -1)
                sk.view(3, -1)[2] = 0.0
        for t in range(T - 1):
            pl = sd[f"products.{t}.linear.weight"].view(3, C * C)
            pl[:2] = md[f"products.{t}.linear.weight"].view(2, C * C)
            pl[2] = 0.0
    return large


class ScaleShiftMACECore(_CoreRepulsion, ScaleShiftMACE):
    """ScaleShiftMACE (0e+1o+2e) with mace's pair_repulsion and distance_transform options (tests/mace_zbl_ref.py)"""

    def __init__(self, atomic_numbers, pair_repulsion=False, distance_transform=None, **kw):
        super().__init__(atomic_numbers, **kw)
        self._add_options(pair_repulsion, distance_transform)


def make_mace_l2_core(seed=0, atomic_numbers=(14, 6, 8), pair_repulsion=True, distance_transform="agnesi", **kw):
    """make_mace_l2 with the ZBL pair term and (by default) the Agnesi transform"""
    return _zbl._make(ScaleShiftMACECore, seed, atomic_numbers, pair_repulsion, distance_transform, kw)
