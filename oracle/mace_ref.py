"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

CPU restatement (torch, float64 by default) of mace's `ScaleShiftMACE` with scalar hidden features
(hidden_irreps = C x 0e, max_L = 0), with mace's attribute tree and state_dict names, and autograd energy / forces /
stress.  This module is the single place where the e3nn / mace conventions the engine relies on are written down.
mace and e3nn are not available here, so every convention below is recalled, not pinned against a mace checkout:

  * spherical harmonics (`sh_basis`): real, `normalize=True`, "component" normalisation (sum_m Y_lm^2 = 2l + 1), in
    the order l = 0..max_ell and inside each l the polynomials listed in `sh_basis`.  The symmetric-contraction
    tensors U are generated in this same basis (`make_u`), so only the pair (SH, U) has to be consistent.
  * edge vector v = r_receiver - r_sender (+ lattice shift); messages are summed at the receiver.
  * radial basis: b_n(d) = prefactor sin(w_n d) / d * f_cut(d / r_max), prefactor = sqrt(2 / r_max), w_n = n pi / r_max
    (`bessel_weights`); f_cut is mace's PolynomialCutoff(p).
  * e3nn FullyConnectedNet: x @ W / sqrt(fan_in) per layer, activation c_act * SiLU between layers (none after the
    last); c_act = e3nn's normalize2mom constant, read from `layer.act.cst`, else `SILU_2MOM`.
  * e3nn Linear between scalar multiplicities: flat weight viewed [C_in, C_out], x @ W / sqrt(C_in); several l blocks
    are concatenated in ascending l.
  * e3nn FullyConnectedTensorProduct with the one-hot element attributes (skip_tp): flat weight viewed
    [C_in, n_elem, C_out] per path (paths in ascending l), divided by sqrt(C_in * n_elem).
  * convolution 0e x Y_l -> l ("uvu"): path constant 1; the radial MLP output is [E, (max_ell + 1) * C], l-major.
  * 1 / avg_num_neighbors is applied to the summed message, before the interaction's `linear`.
  * symmetric contraction: B[c] = sum_nu sum_k w_nu[z, k, c] sum_{i1..inu} U_nu[i1..inu, k] A[c, i1] ... A[c, inu];
    `weights_max` belongs to nu = correlation, `weights.{j}` to nu = correlation - 1 - j.
  * readouts: LinearReadoutBlock h @ w / sqrt(C); NonLinearReadoutBlock (c_act SiLU(h @ W1 / sqrt(C))) @ W2 / sqrt(H).
  * energy of atom i: E0[z_i] + scale * sum_t e_t(i) + shift; stress = dE/d(strain) / V (symmetric strain).
  * e3nn's bookkeeping buffers (`*.output_mask`, all ones; the empty `weight` of a TensorProduct fed external weights)
    may appear in a mace state_dict; they carry no arithmetic, so this tree does not register them and the engine accepts
    and checks them.
"""
from __future__ import annotations

import functools
import itertools
import math

import numpy as np
import torch
from torch import nn

# e3nn normalize2mom(SiLU): 1 / sqrt(E[SiLU(z)^2]), z ~ N(0, 1), by quadrature (e3nn estimates it by sampling)
SILU_2MOM = 1.6765324703310909


def nsh_of(max_ell):
    return (max_ell + 1) ** 2


def l_of_index(max_ell):
    return [l for l in range(max_ell + 1) for _ in range(2 * l + 1)]


def sh_basis(vec, max_ell):
    """[E, 3] edge vectors -> [E, (max_ell+1)^2] real spherical harmonics of the unit vector, component-normalised."""
    r = vec / torch.linalg.norm(vec, dim=-1, keepdim=True)
    x, y, z = r[..., 0], r[..., 1], r[..., 2]
    out = [torch.ones_like(x)]
    if max_ell >= 1:
        s3 = math.sqrt(3.0)
        out += [s3 * x, s3 * y, s3 * z]
    if max_ell >= 2:
        s15, s5 = math.sqrt(15.0), math.sqrt(5.0)
        out += [s15 * x * y, s15 * y * z, 0.5 * s5 * (2 * z * z - x * x - y * y), s15 * x * z, 0.5 * s15 * (x * x - y * y)]
    if max_ell >= 3:
        a, b, c, d = math.sqrt(70.0) / 4, math.sqrt(105.0), math.sqrt(42.0) / 4, math.sqrt(7.0) / 2
        q = 4 * z * z - x * x - y * y
        out += [a * y * (3 * x * x - y * y), b * x * y * z, c * y * q, d * z * (2 * z * z - 3 * x * x - 3 * y * y),
                c * x * q, 0.5 * b * z * (x * x - y * y), a * x * (x * x - 3 * y * y)]
    if max_ell > 3:
        raise NotImplementedError("max_ell <= 3")
    return torch.stack(out, dim=-1)


def polynomial_cutoff(d, r_max, p):
    x = d / r_max
    f = (1.0 - 0.5 * (p + 1) * (p + 2) * x ** p + p * (p + 2) * x ** (p + 1) - 0.5 * p * (p + 1) * x ** (p + 2))
    return f * (x < 1.0)


# ------------------------------------------------------------------------------------------ U tensors
def wigner_d(rot, max_ell, rng):
    """Real Wigner-D of a 3x3 orthogonal matrix in the basis of `sh_basis`: Y(rot r) = D Y(r), fitted on points."""
    pts = torch.tensor(rng.normal(size=(400, 3)), dtype=torch.float64)
    y0 = sh_basis(pts, max_ell)
    y1 = sh_basis(pts @ torch.as_tensor(rot, dtype=torch.float64).T, max_ell)
    return torch.linalg.lstsq(y0, y1).solution.T  # y1 = y0 D^T


def _random_rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


@functools.lru_cache(maxsize=None)
def make_u(max_ell, nu, seed=0):
    """Orthonormal basis of the permutation-symmetric, O(3)-invariant tensors of order nu over (+)_{l<=max_ell} Y_l:
    the null space of D(g)^{(x)nu} - I on the symmetric subspace, g in {two random rotations, inversion}.
    Returns [nsh]*nu + [K] float64."""
    rng = np.random.default_rng(seed)
    n = nsh_of(max_ell)
    gens = [wigner_d(_random_rotation(rng), max_ell, rng) for _ in range(2)]
    gens.append(torch.diag(torch.tensor([(-1.0) ** l for l in l_of_index(max_ell)], dtype=torch.float64)))
    lidx = l_of_index(max_ell)
    # D is block-diagonal in l, so the invariants split by the sorted l-tuple of the indices: one null space per
    # tuple keeps every basis tensor inside one block (few nonzeros per tensor; the engine evaluates U sparsely)
    by_l = {}
    for ms in itertools.combinations_with_replacement(range(n), nu):
        by_l.setdefault(tuple(lidx[i] for i in ms), []).append(ms)
    out = []
    for key in sorted(by_l):
        multisets = by_l[key]
        S = torch.zeros(len(multisets), *([n] * nu), dtype=torch.float64)
        for m, ms in enumerate(multisets):
            for perm in set(itertools.permutations(ms)):
                S[(m,) + perm] = 1.0
        S = S / torch.linalg.norm(S.reshape(len(multisets), -1), dim=1).reshape(-1, *([1] * nu))
        blocks = []
        for D in gens:
            T = S
            for ax in range(nu):
                T = torch.movedim(torch.tensordot(T, D, dims=([1 + ax], [1])), -1, 1 + ax)
            blocks.append((T - S).reshape(len(multisets), -1))
        Uv, sv, _ = torch.linalg.svd(torch.cat(blocks, dim=1), full_matrices=False)
        sv_full = torch.zeros(len(multisets), dtype=torch.float64)
        sv_full[: len(sv)] = sv
        null = Uv[:, sv_full < 1e-9]  # [n_multisets, K_block]
        out.append(torch.tensordot(null, S, dims=([0], [0])))  # [K_block, n, ..., n]
    return torch.movedim(torch.cat(out, dim=0), 0, -1).contiguous()


# ------------------------------------------------------------------------------------------ modules
class _Act(nn.Module):
    """e3nn normalize2mom(SiLU): `cst` is a plain attribute, as the engine's wrapper reads it"""

    def __init__(self, cst=SILU_2MOM):
        super().__init__()
        self.cst = cst

    def forward(self, x):
        return self.cst * torch.nn.functional.silu(x)


class _FCLayer(nn.Module):
    def __init__(self, h_in, h_out, act):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(h_in, h_out, dtype=torch.float64))
        self.act = _Act() if act else None

    def forward(self, x):
        x = x @ (self.weight / math.sqrt(self.weight.shape[0]))
        return self.act(x) if self.act is not None else x


class FullyConnectedNet(nn.Module):
    def __init__(self, hs):
        super().__init__()
        for k in range(len(hs) - 1):
            setattr(self, f"layer{k}", _FCLayer(hs[k], hs[k + 1], k < len(hs) - 2))
        self.hs = list(hs)

    def forward(self, x):
        for k in range(len(self.hs) - 1):
            x = getattr(self, f"layer{k}")(x)
        return x


class _W(nn.Module):
    """a module holding only a flat e3nn `weight`"""

    def __init__(self, numel, scale=1.0):
        super().__init__()
        self.weight = nn.Parameter(scale * torch.randn(numel, dtype=torch.float64))


class BesselBasis(nn.Module):
    def __init__(self, r_max, num_basis):
        super().__init__()
        self.register_buffer("bessel_weights", math.pi / r_max * torch.arange(1, num_basis + 1, dtype=torch.float64))
        self.register_buffer("r_max", torch.tensor(float(r_max), dtype=torch.float64))
        self.register_buffer("prefactor", torch.tensor(math.sqrt(2.0 / r_max), dtype=torch.float64))

    def forward(self, d):  # [E, 1]
        return self.prefactor * torch.sin(self.bessel_weights * d) / d


class PolynomialCutoff(nn.Module):
    def __init__(self, r_max, p):
        super().__init__()
        self.register_buffer("p", torch.tensor(float(p), dtype=torch.float64))
        self.register_buffer("r_max", torch.tensor(float(r_max), dtype=torch.float64))

    def forward(self, d):
        return polynomial_cutoff(d, self.r_max, self.p)


class RadialEmbeddingBlock(nn.Module):
    def __init__(self, r_max, num_bessel, p):
        super().__init__()
        self.bessel_fn = BesselBasis(r_max, num_bessel)
        self.cutoff_fn = PolynomialCutoff(r_max, p)

    def forward(self, d):
        return self.bessel_fn(d) * self.cutoff_fn(d)


class LinearNodeEmbeddingBlock(nn.Module):
    def __init__(self, n_elem, C):
        super().__init__()
        self.linear = _W(n_elem * C)
        self.n_elem, self.C = n_elem, C

    def forward(self, z):
        return self.linear.weight.view(self.n_elem, self.C)[z] / math.sqrt(self.n_elem)


class _Interaction(nn.Module):
    def __init__(self, C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors, residual):
        super().__init__()
        self.C, self.n_elem, self.max_ell, self.residual = C, n_elem, max_ell, residual
        self.avg_num_neighbors = float(avg_num_neighbors)
        L1 = max_ell + 1
        self.linear_up = _W(C * C)
        self.conv_tp_weights = FullyConnectedNet([num_bessel] + list(radial_mlp) + [L1 * C])
        self.linear = _W(L1 * C * C)
        self.skip_tp = _W((1 if residual else L1) * C * n_elem * C)

    def forward(self, h, z, Y, ef, src, dst):
        C, n, L1 = self.C, h.shape[0], self.max_ell + 1
        lsel = torch.tensor(l_of_index(self.max_ell))
        u = h @ self.linear_up.weight.view(C, C) / math.sqrt(C)
        R = self.conv_tp_weights(ef).view(-1, L1, C)[:, lsel, :]  # [E, nsh, C]
        m = u[src][:, None, :] * R * Y[:, :, None]
        A = torch.zeros(n, Y.shape[1], C, dtype=h.dtype).index_add(0, dst, m) / self.avg_num_neighbors
        Wl = self.linear.weight.view(L1, C, C)[lsel] / math.sqrt(C)  # [nsh, C, C]
        A = torch.einsum("nic,icd->nid", A, Wl)
        norm = math.sqrt(C * self.n_elem)
        if self.residual:
            Ws = self.skip_tp.weight.view(C, self.n_elem, C)
            sc = torch.einsum("nc,ncd->nd", h, Ws.permute(1, 0, 2)[z]) / norm
            return A, sc
        Ws = self.skip_tp.weight.view(L1, C, self.n_elem, C)[lsel]  # [nsh, C, n_elem, C]
        A = torch.einsum("nic,nicd->nid", A, Ws.permute(2, 0, 1, 3)[z]) / norm
        return A, None


class RealAgnosticResidualInteractionBlock(_Interaction):
    def __init__(self, *a):
        super().__init__(*a, residual=True)


class RealAgnosticInteractionBlock(_Interaction):
    def __init__(self, *a):
        super().__init__(*a, residual=False)


class Contraction(nn.Module):
    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.correlation = correlation
        for nu in range(1, correlation + 1):
            self.register_buffer(f"U_matrix_{nu}", make_u(max_ell, nu).clone())
        K = lambda nu: getattr(self, f"U_matrix_{nu}").shape[-1]
        self.weights_max = nn.Parameter(torch.randn(n_elem, K(correlation), C, dtype=torch.float64) / K(correlation))
        self.weights = nn.ParameterList(
            [nn.Parameter(torch.randn(n_elem, K(nu), C, dtype=torch.float64) / K(nu)) for nu in range(correlation - 1, 0, -1)])

    def weight_of(self, nu):
        return self.weights_max if nu == self.correlation else self.weights[self.correlation - 1 - nu]

    def forward(self, A, z):  # A [n, nsh, C]
        B = torch.zeros(A.shape[0], A.shape[2], dtype=A.dtype)
        for nu in range(1, self.correlation + 1):
            U = getattr(self, f"U_matrix_{nu}")
            nz = U.nonzero(as_tuple=True)  # U is sparse (one l-tuple per basis tensor): sum over its nonzeros
            prod = U[nz][None, :, None] * A[:, nz[0], :]
            for j in range(1, nu):
                prod = prod * A[:, nz[j], :]
            P = torch.zeros(A.shape[0], U.shape[-1], A.shape[2], dtype=A.dtype).index_add(1, nz[nu], prod)
            B = B + (self.weight_of(nu)[z] * P).sum(dim=1)
        return B


class SymmetricContraction(nn.Module):
    def __init__(self, *a):
        super().__init__()
        self.contractions = nn.ModuleList([Contraction(*a)])

    def forward(self, A, z):
        return self.contractions[0](A, z)


class EquivariantProductBasisBlock(nn.Module):
    def __init__(self, max_ell, correlation, n_elem, C):
        super().__init__()
        self.symmetric_contractions = SymmetricContraction(max_ell, correlation, n_elem, C)
        self.linear = _W(C * C)
        self.C = C

    def forward(self, A, sc, z):
        h = self.symmetric_contractions(A, z) @ self.linear.weight.view(self.C, self.C) / math.sqrt(self.C)
        return h + sc if sc is not None else h


class LinearReadoutBlock(nn.Module):
    def __init__(self, C):
        super().__init__()
        self.linear = _W(C)

    def forward(self, h):
        return h @ self.linear.weight / math.sqrt(h.shape[1])


class NonLinearReadoutBlock(nn.Module):
    def __init__(self, C, H):
        super().__init__()
        self.linear_1 = _W(C * H)
        self.non_linearity = _Act()
        self.linear_2 = _W(H)
        self.C, self.H = C, H

    def forward(self, h):
        x = self.non_linearity(h @ self.linear_1.weight.view(self.C, self.H) / math.sqrt(self.C))
        return x @ self.linear_2.weight / math.sqrt(self.H)


class ScaleShiftBlock(nn.Module):
    def __init__(self, scale, shift):
        super().__init__()
        self.register_buffer("scale", torch.tensor(float(scale), dtype=torch.float64))
        self.register_buffer("shift", torch.tensor(float(shift), dtype=torch.float64))


class AtomicEnergiesBlock(nn.Module):
    def __init__(self, e0):
        super().__init__()
        self.register_buffer("atomic_energies", torch.as_tensor(e0, dtype=torch.float64))


class ScaleShiftMACE(nn.Module):
    """mace.modules.ScaleShiftMACE restricted to hidden_irreps = C x 0e (the engine's supported configuration)."""

    def __init__(self, atomic_numbers, C=32, max_ell=3, correlation=3, num_interactions=2, r_max=5.0, num_bessel=8,
                 num_polynomial_cutoff=5, radial_mlp=(64, 64, 64), avg_num_neighbors=20.0, mlp_hidden=16,
                 interaction_classes=None, scale=1.0, shift=0.0, atomic_energies=None):
        super().__init__()
        n_elem = len(atomic_numbers)
        self.register_buffer("atomic_numbers", torch.as_tensor(atomic_numbers, dtype=torch.int64))
        self.register_buffer("r_max", torch.tensor(float(r_max), dtype=torch.float64))
        self.register_buffer("num_interactions", torch.tensor(int(num_interactions), dtype=torch.int64))
        self.heads = ["default"]
        self.max_ell, self.correlation = max_ell, correlation
        self.node_embedding = LinearNodeEmbeddingBlock(n_elem, C)
        self.radial_embedding = RadialEmbeddingBlock(r_max, num_bessel, num_polynomial_cutoff)
        if interaction_classes is None:
            interaction_classes = [RealAgnosticInteractionBlock] + [RealAgnosticResidualInteractionBlock] * (num_interactions - 1)
        self.interactions = nn.ModuleList(
            [cls(C, n_elem, max_ell, num_bessel, radial_mlp, avg_num_neighbors) for cls in interaction_classes])
        self.products = nn.ModuleList(
            [EquivariantProductBasisBlock(max_ell, correlation, n_elem, C) for _ in range(num_interactions)])
        self.readouts = nn.ModuleList(
            [LinearReadoutBlock(C) for _ in range(num_interactions - 1)] + [NonLinearReadoutBlock(C, mlp_hidden)])
        self.scale_shift = ScaleShiftBlock(scale, shift)
        e0 = np.zeros(n_elem) if atomic_energies is None else atomic_energies
        self.atomic_energies_fn = AtomicEnergiesBlock(e0)

    def node_energies(self, vec, src, dst, z, taps=None):
        """(eps_i [n], interaction part e_i [n]) for edges (src -> dst) with vectors vec = r_dst - r_src + shift"""
        d = torch.linalg.norm(vec, dim=1, keepdim=True)
        Y = sh_basis(vec, self.max_ell)
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


def species_index(model, atoms):
    zt = {int(a): k for k, a in enumerate(model.atomic_numbers.tolist())}
    return torch.as_tensor([zt[int(a)] for a in atoms.get_atomic_numbers()], dtype=torch.int64)


def potential_ref(model, atoms, calc_forces=True, calc_stresses=True, dtype=torch.float64, taps=None):
    """Energy [1], forces [N, 3] (eV/A) and stress [3, 3] (GPa, dE/d(strain) / V as the engine reports it), plus the
    per-atom energies eps_i, by autograd on the global graph."""
    from oracle.graph_ref import neighbor_list

    lattice_np = np.array(atoms.get_cell())
    cart = np.array(atoms.get_positions(wrap=False))
    pbc = atoms.get_pbc().astype(np.int64)
    i1, i2, off, _d2, _b = neighbor_list(cart, lattice_np, pbc, float(model.r_max), 0.0)
    model = model.to(dtype)
    lattice = torch.tensor(lattice_np, dtype=dtype)
    strain = torch.zeros(3, 3, dtype=dtype, requires_grad=True)
    sym = 0.5 * (strain + strain.T)
    pos0 = torch.tensor(cart, dtype=dtype, requires_grad=True)
    pos = pos0 @ (torch.eye(3, dtype=dtype) + sym)
    lat = lattice @ (torch.eye(3, dtype=dtype) + sym)
    t = lambda a: torch.as_tensor(a, dtype=torch.int64)
    vec = pos[t(i2)] + torch.tensor(off, dtype=dtype) @ lat - pos[t(i1)]
    z = species_index(model, atoms)
    eps, _ = model.node_energies(vec, t(i1), t(i2), z, taps=taps)
    total = eps.sum()
    forces = stress = None
    if calc_forces or calc_stresses:
        gp, gs = torch.autograd.grad(total, (pos0, strain))
        forces = -gp
        vol = abs(np.linalg.det(lattice_np))
        stress = gs / vol * 160.21766208
    return total.detach().reshape(1), forces, stress, eps.detach()


def atomic_virials_ref(model, atoms, dtype=torch.float64):
    """Per-atom virials [N, 3, 3] (eV) by autograd: w_i = 1/2 sum over the edges e with endpoint i of v_e (x) dE/dv_e,
    the edge vectors v_e being leaves of the graph (the engine's b2m_get_atomic convention)."""
    from oracle.graph_ref import neighbor_list

    lattice_np = np.array(atoms.get_cell())
    cart = np.array(atoms.get_positions(wrap=False))
    i1, i2, off, _d2, _b = neighbor_list(cart, lattice_np, atoms.get_pbc().astype(np.int64), float(model.r_max), 0.0)
    model = model.to(dtype)
    src, dst = torch.as_tensor(i1, dtype=torch.int64), torch.as_tensor(i2, dtype=torch.int64)
    pos = torch.tensor(cart, dtype=dtype)
    vec = (pos[dst] + torch.tensor(off, dtype=dtype) @ torch.tensor(lattice_np, dtype=dtype) - pos[src]).requires_grad_()
    eps, _ = model.node_energies(vec, src, dst, species_index(model, atoms))
    g, = torch.autograd.grad(eps.sum(), vec)
    half = 0.5 * vec.detach()[:, :, None] * g[:, None, :]
    w = torch.zeros(len(atoms), 3, 3, dtype=dtype)
    return w.index_add(0, src, half).index_add(0, dst, half)


def make_mace(seed=0, atomic_numbers=(14, 6, 8), **kw):
    """seeded random ScaleShiftMACE (weights N(0, 1), as e3nn initialises them)"""
    torch.manual_seed(seed)
    kw.setdefault("atomic_energies", np.linspace(-3.0, -1.0, len(atomic_numbers)))
    kw.setdefault("scale", 1.3)
    kw.setdefault("shift", -0.2)
    return ScaleShiftMACE(list(atomic_numbers), **kw)
