"""Kernel-unit tests of the MACE path: input generators and a float64 restatement of every launcher of kernels_mace.cu
with a per-element error scale, in the manner of tests/kernel_units_ref.py (whose `Mag`, `max_err` and shim it uses).

Conventions are not restated here: harmonics, Bessel basis and cutoff come from oracle/mace_ref.py, the conv_tp paths
and coupling tensors from tests/mace_eq_ref.py, the symmetric contraction from the contraction modules of both (their
forward, on U and weights rounded to fp32, is the reference, so the host term builder is under test too), ZBL and
Agnesi from tests/mace_zbl_ref.py.

Scales, in units of one fp32 rounding of the quantity they sit beside:
  * multilinear launchers (messages, element mixes, contractions, linear readouts and their reverses): the same
    operation on |inputs| and |coefficients|, i.e. the sum of the absolute values of the terms; the reverse scales are
    the gradients of that absolute forward against |upstream|;
  * per-edge functions of the fp32 edge vector (harmonics, radial basis, ZBL, the final geometry reverse):
    |q| + sum_i |dq/dv_i| |v_i| (the input's rounding carried through; for the sin argument w_n d up to 64 pi this is
    the term w_n |cos| that the argument's rounding costs; the Agnesi argument x adds |db/dx| 3 x), plus, where `__powf` evaluates the polynomial envelope, its
    powers times (2 + (p - 1) (3 + |log2 x|)) (lg2 / ex2 approximations);
  * SiLU and SiLU' through `__expf`: the argument carries 2 + 1.5 |x| (ex2.approx of x log2 e);
  * sums accumulated in double (readout_final's energy, the virial) add 2^-29 |x| per term.
Values of reverse launchers come from torch.autograd of the forward restatement.
"""
from __future__ import annotations

import copy
import ctypes
import math

import torch

from oracle import mace_ref as MR
from tests import mace_eq_ref as EQ
from tests import mace_zbl_ref as ZR
from tests.kernel_units_ref import F64, SENTINEL, Mag, d64

# |out - ref| <= TOL * scale, per element.  Set from the H100 run recorded in DESIGN.md section 5 (at least 3x the
# largest error observed) and at least 10x below every mutant (tests/test_mace_units_cpu.py).
TOL = {"edge_geom": 1e-6, "zbl": 3e-7, "msg": 7e-7, "msg_bwd": 7e-7, "msg_eq": 1e-6, "msg_eq_bwd": 1e-6,
       "elem_mix": 1e-6, "symc": 3e-6, "symc_bwd": 3e-6, "readout": 5e-7, "edge_final": 4e-7}
DBL = 2.0 ** -29  # one double rounding, in units of an fp32 one
R_MAX, P_CUT = 5.0, 5
ELEMS = (1, 8, 26)  # atomic numbers of the element table (H, O, Fe: far apart in Z and radius)


def f32(t):
    return t.float().to(F64)


# ------------------------------------------------------------------------------------------------ model constants
def radial_params(nb):
    """(w [nb] fp32, prefactor) of mace's Bessel basis (oracle/mace_ref.py BesselBasis) at R_MAX"""
    b = MR.BesselBasis(R_MAX, nb)
    return b.bessel_weights.float(), float(b.prefactor)


def core_params(zbl, agnesi):
    """element table [n_elem][4] fp32 (Z, Z^a_exp, ZBL radius, Agnesi radius), cf (za, zc[4], zscale, aq, ap, aa),
    zp, and the float64 modules (tests/mace_zbl_ref.py)"""
    zb, ag = ZR.ZBLBasis(), ZR.AgnesiTransform()
    Z = torch.tensor(ELEMS, dtype=F64)
    tab = torch.stack([Z, Z ** zb.a_exp, zb.covalent_radii[list(ELEMS)], ag.covalent_radii[list(ELEMS)]], 1).float()
    cf = torch.tensor([float(zb.a_prefactor) * 0.529] + zb.c.tolist() + [1.3, float(ag.q), float(ag.p), float(ag.a)],
                      dtype=torch.float32)
    return dict(elem=tab, cf=cf, zp=int(zb.p), zbl=int(zbl), agnesi=int(agnesi), zb=zb, ag=ag, zscale=1.3)


# ------------------------------------------------------------------------------------------------ graphs
def gen_graph(n_own, seed, n_halo=None, empty=0, heavy=0, per_row=6, close=True, E=None):
    """One partition's CSR-by-destination graph: e_dst ascending over n_own owned atoms (`empty` of them without
    edges, one with `heavy` edges), e_src over n_loc = n_own + n_halo rows with a quarter of the sources in the halo,
    types mixed, gid a permutation of N = n_own + 3 global ids (halo rows images of random atoms, one halo row the
    image of an edge's own destination: a self-image edge), E edges over the rows when E is given, |e_vec.xyz| = e_vec.w in fp32 with distances in
    [0.3, R_MAX) (a few within 1e-4 A of R_MAX, close contacts down to 0.3 A)."""
    g = torch.Generator().manual_seed(seed)
    n_halo = max(2, n_own // 3) if n_halo is None else n_halo
    n_loc, N = n_own + n_halo, n_own + 3
    cnt = torch.randint(1, 2 * per_row, (n_own,), generator=g)
    if n_own:
        cnt[torch.randperm(n_own, generator=g)[:empty]] = 0
        if heavy:
            cnt[int(torch.randint(0, n_own, (1,), generator=g))] = heavy
    if E is not None:
        rows = torch.nonzero(cnt > 0).flatten()
        cnt = torch.bincount(rows[torch.randint(0, len(rows), (E,), generator=g)], minlength=n_own)
    E = int(cnt.sum())
    row_ptr = torch.cat([torch.zeros(1, dtype=torch.long), cnt.cumsum(0)]).int()
    dst = torch.repeat_interleave(torch.arange(n_own), cnt).int()
    src = torch.randint(0, n_loc, (E,), generator=g)
    if E > 3:
        sel = torch.randperm(E, generator=g)[: E // 4]
        src[sel] = torch.randint(n_own, n_loc, (len(sel),), generator=g)
    type_ = torch.randint(0, len(ELEMS), (n_loc,), generator=g).int()
    gid = torch.empty(n_loc, dtype=torch.long)
    gid[:n_own] = torch.randperm(N, generator=g)[:n_own]
    gid[n_own:] = gid[:n_own][torch.randint(0, max(n_own, 1), (n_halo,), generator=g)] if n_own else 0
    if E:  # self-image edge: a halo source with the gid (and species) of the edge's destination
        e0 = int(torch.randint(0, E, (1,), generator=g))
        h = n_own + int(torch.randint(0, n_halo, (1,), generator=g))
        src[e0] = h
        gid[h], type_[h] = gid[dst[e0].long()], type_[dst[e0].long()]
    d = 0.9 + (R_MAX - 0.9) * torch.rand(E, generator=g, dtype=F64)
    if E:
        nc = torch.randperm(E, generator=g)[: max(1, E // 16)]
        d[nc] = R_MAX - 1e-4 * torch.rand(len(nc), generator=g, dtype=F64)
        if close:
            cc = torch.randperm(E, generator=g)[: max(1, E // 8)]
            d[cc] = 0.3 + 0.9 * torch.rand(len(cc), generator=g, dtype=F64)
    u = torch.randn(E, 3, generator=g, dtype=F64)
    u = u / u.norm(dim=1, keepdim=True)
    xyz = (u * d[:, None]).float()
    e_vec = torch.cat([xyz, xyz.to(F64).norm(dim=1, keepdim=True).float()], 1)
    return dict(n_own=n_own, n_loc=n_loc, N=N, E=E, row_ptr=row_ptr, e_src=src.int(), e_dst=dst, e_vec=e_vec,
                type=type_, gid=gid.int(), g=g)


def restrict(c, n):
    """the graph of the first n owned rows (their edges, the same local rows)"""
    E = int(c["row_ptr"][n])
    r = dict(c, n_own=n, E=E, row_ptr=c["row_ptr"][: n + 1].clone())
    for k in ("e_src", "e_dst", "e_vec"):
        r[k] = c[k][:E]
    return r


def rnd(g, *shape, s=1.0, Cr=None):
    """unit-scale random fp32 [.., C] with channels >= Cr zero (the padding of the row pitch)"""
    x = torch.randn(*shape, generator=g) * s
    if Cr is not None:
        x[..., Cr:] = 0.0
    return x


def plus(prefill, x, s=None):
    """prefill + x as a Mag (x a Mag, or a value with scale s)"""
    if isinstance(x, Mag):
        x, s = x.x, x.s
    p = d64(prefill)
    return Mag(p + x.reshape(p.shape), p.abs() + s.reshape(p.shape))


def flat(m):
    return Mag(m.x.reshape(-1), m.s.reshape(-1))


def KU_mag(m, shape):
    return Mag(m.x.reshape(shape), m.s.reshape(shape))


def symc_terms_fwd(terms, A, w, z, eq, nsh):
    """B [(4 or 1)][n][C] walked over the term list in float64 (the host builder's terms, not U)"""
    A, w = d64(A), d64(w)
    n, C = A.shape[1], A.shape[2]
    B = torch.zeros(4 if eq else 1, n, C, dtype=F64)
    coef = d64(terms[:, 2].contiguous().view(torch.float32))
    for j in range(len(terms)):
        t = int(terms[j, 0])
        nu, o = (t >> 24) & 3, (t >> 28) & 3
        prod = coef[j] * w[z, int(terms[j, 1])]
        for i in [t & 255, (t >> 8) & 255, (t >> 16) & 255][:nu]:
            prod = prod * A[i]
        B[o] += prod
    return B


# ------------------------------------------------------------------------------------------------ scale helpers
def _jvp_cols(f, x, cols):
    """[dy/dx_j for j in cols] of a row-wise f, by forward mode"""
    out = []
    for j in cols:
        t = torch.zeros_like(x)
        t[:, j] = 1.0
        out.append(torch.func.jvp(f, (x,), (t,))[1])
    return out


def powf_rel(x, p):
    """relative error scale of x^k evaluated with __powf (lg2 / ex2 approximations), 0 where x >= 1"""
    x = x.clamp(1e-30, 1.0)
    return torch.where(x < 1.0, 2.0 + (p - 1) * (3.0 + torch.log2(x).abs()), torch.zeros_like(x))


def env_powf_scale(x, p):
    """|powers of the envelope| times their __powf relative error (f), and the same for df (times r)"""
    rel = powf_rel(x, p)
    xp = x.clamp(0, 1) ** p
    sf = (0.5 * (p + 1) * (p + 2) * xp + p * (p + 2) * xp * x + 0.5 * p * (p + 1) * xp * x * x) * rel
    sdf = (0.5 * (p + 1) * (p + 2) * p * xp / x.clamp_min(1e-30) + p * (p + 2) * (p + 1) * xp
           + 0.5 * p * (p + 1) * (p + 2) * xp * x) * rel
    return sf, sdf


def silu_scale(x, s_in):
    """Mag of silu(x) with the __expf rounding of its argument"""
    return Mag(x, s_in + 2.0 + 1.5 * x.abs()).apply(torch.nn.functional.silu)


def dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


# ------------------------------------------------------------------------------------------------ edge geometry
def sh(v, nsh, mut=()):
    """[E][16] harmonics (oracle/mace_ref.py sh_basis) of max_ell = sqrt(nsh) - 1, zero past nsh"""
    Y = MR.sh_basis(v, int(round(math.sqrt(nsh))) - 1)
    if "y_swap_11_13" in mut and nsh == 16:
        Y = Y[:, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 13, 12, 11, 14, 15]]
    return torch.cat([Y, torch.zeros(len(v), 16 - nsh, dtype=Y.dtype)], 1)


def zn(c, core):
    Z = torch.tensor(ELEMS, dtype=torch.long)
    return Z[c["type"].long()[c["e_src"].long()]], Z[c["type"].long()[c["e_dst"].long()]]


def bessel(d, c, nb, core):
    """b_n(x) [E][nb] without the cutoff (the factor the envelope's rounding multiplies)"""
    x = d[:, None]
    if core["agnesi"]:
        Zu, Zv = zn(c, core)
        x = core["ag"](d[:, None], Zu, Zv)
    return MR.BesselBasis(R_MAX, nb)(x)


def radial_basis(d, c, nb, core, mut=()):
    """eb [E][64]: b_n(x) f_cut(d), x = d or Agnesi's x(d, Z_src, Z_dst); d [E] float64"""
    bes = MR.BesselBasis(R_MAX, nb)
    x = d[:, None]
    if core["agnesi"]:
        Zu, Zv = zn(c, core)
        x = core["ag"](d[:, None], Zu, Zv)
        if "no_agnesi_dx" in mut:
            x = x.detach() + (d - d.detach())[:, None]
    f = MR.polynomial_cutoff(d, R_MAX, P_CUT)[:, None]
    if "no_env_df" in mut:
        f = f.detach()
    b = bes(x) * f
    if "no_last_bessel" in mut:
        b = torch.cat([b[:, :-1], torch.zeros_like(b[:, -1:])], 1)
    return torch.cat([b, torch.zeros(len(d), 64 - nb, dtype=b.dtype)], 1)


def edge_geom_ref(c, nb, nsh, core, mut=()):
    """{Y, eb}: Mags [E][16], [E][64]"""
    v, d = d64(c["e_vec"][:, :3]), d64(c["e_vec"][:, 3])
    Y = sh(v, nsh, mut)
    dY = _jvp_cols(lambda x: sh(x, nsh), v, range(3))
    sY = Y.abs() + sum(dY[j].abs() * v[:, j:j + 1].abs() for j in range(3))
    eb = radial_basis(d, c, nb, core, mut)
    deb = torch.func.jvp(lambda x: radial_basis(x, c, nb, core), (d,), (d,))[1]  # d eb/dd * d
    bes = torch.nn.functional.pad(bessel(d, c, nb, core), (0, 64 - nb))
    sf, _ = env_powf_scale(d / R_MAX, P_CUT)
    seb = eb.abs() + deb.abs() + bes.abs() * sf[:, None]
    if core["agnesi"]:  # x = 1 + a s^q / (1 + s^(q - p)) carries a few roundings of x itself, more than dx/dd d
        Zu, Zv = zn(c, core)
        x = core["ag"](d[:, None], Zu, Zv)
        f = MR.polynomial_cutoff(d, R_MAX, P_CUT)[:, None]
        dbx = torch.func.jvp(lambda t: MR.BesselBasis(R_MAX, nb)(t) * f, (x,), (3.0 * x,))[1]
        seb = seb + torch.nn.functional.pad(dbx.abs(), (0, 64 - nb))
    return dict(Y=Mag(Y, sY), eb=Mag(eb, seb))


def zbl_edge(d, c, core):
    Zu, Zv = zn(c, core)
    return core["zb"].edge_energies(d, Zu, Zv)


def zbl_ref(c, core, e_lin):
    """e_lin (owned rows) += the ZBL energies of the edges into each row"""
    d = d64(c["e_vec"][:, 3])
    V = zbl_edge(d, c, core)
    dV = torch.func.jvp(lambda x: zbl_edge(x, c, core), (d,), (d,))[1]
    Zu, Zv = zn(c, core)
    rc = core["zb"].covalent_radii[Zu] + core["zb"].covalent_radii[Zv]
    far = copy.deepcopy(core["zb"])  # the pair term without its envelope (a cutoff far away)
    far.covalent_radii.mul_(1e9)
    sf, _ = env_powf_scale(d / rc, core["zp"])
    s = V.abs() + dV.abs() + far.edge_energies(d, Zu, Zv).abs() * sf
    dst = c["e_dst"].long()
    x = d64(e_lin).index_add(0, dst, V)
    return Mag(x, d64(e_lin).abs().index_add(0, dst, s))


# ------------------------------------------------------------------------------------------------ multilinear ops
def multilinear(f, xs, g=None, wrt=()):
    """value and scale of f(*xs) (f multilinear in xs, `absolute` flag taking |coefficients|), and, with upstream g,
    {name: Mag} of d(f . g)/dx for x in wrt (values by autograd, scales by autograd of the absolute forward)."""
    xs = {k: d64(v) for k, v in xs.items()}
    ax = {k: v.abs() for k, v in xs.items()}
    if g is None:
        with torch.no_grad():
            return Mag(f(False, **xs), f(True, **ax))
    xs = {k: v.requires_grad_(k in wrt) for k, v in xs.items()}
    ax = {k: v.requires_grad_(k in wrt) for k, v in ax.items()}
    with torch.enable_grad():
        y = f(False, **xs)
        gv = torch.autograd.grad((y * d64(g)).sum(), [xs[k] for k in wrt])
        ya = f(True, **ax)
        gs = torch.autograd.grad((ya * d64(g).abs()).sum(), [ax[k] for k in wrt])
    out = {k: Mag(gv[i], gs[i]) for i, k in enumerate(wrt)}
    out["_y"] = Mag(y.detach(), ya.detach())
    return out


def l_sel(nsh):
    return torch.tensor(MR.l_of_index(int(round(math.sqrt(nsh))) - 1))


def msg_fn(c, C, L1, mut=()):
    """A [nsh][n_own][C] of k_mace_msg from R [E][L1 C], Y [E][16], u [n_loc][C]"""
    nsh, src, dst = L1 * L1, c["e_src"].long(), c["e_dst"].long()
    ls = l_sel(nsh)

    def f(absolute, R, Y, u):
        Rl = R.view(-1, L1, C)[:, ls, :]  # [E][nsh][C]
        m = Rl * Y[:, :nsh, None] * u[src][:, None, :]
        return torch.zeros(c["n_own"], nsh, C, dtype=F64).index_add(0, dst, m).permute(1, 0, 2)
    return f


def eq_layout(max_ell):
    """conv_tp paths (tests/mace_eq_ref.py), per l_out the path indices, and the slot base of each l_out block"""
    paths = EQ.conv_paths(max_ell, 1)
    per = [[p for p, pt in enumerate(paths) if pt[2] == l] for l in range(max_ell + 1)]
    base, b = [], 0
    for l in range(max_ell + 1):
        base.append(b)
        b += (2 * l + 1) * len(per[l])
    return paths, per, base, b


def msg_eq_fn(c, C, max_ell, mut=()):
    """Am (flat, the slot layout of mace_state.cuh) of k_mace_msg_eq from R [E][NP][C], Y [E][16], u [n_loc][4][C]"""
    paths, per, base, nslots = eq_layout(max_ell)
    src, dst, n = c["e_src"].long(), c["e_dst"].long(), c["n_own"]
    NP = len(paths)
    flip = next(p for p, pt in enumerate(paths) if 3 in pt[1:]) if max_ell == 3 else None

    def cg_of(p, absolute):
        li, ls, lo = paths[p]
        cg = EQ.make_cg(li, ls, lo).clone()
        if "no_sqrt_2l1" not in mut:
            cg = cg * math.sqrt(2 * lo + 1)
        if "cg_sign_l3" in mut and p == flip:
            i = tuple(int(a) for a in torch.nonzero(cg.abs() > 1e-6)[0])
            cg[i] = -cg[i]
        return cg.abs() if absolute else cg

    def f(absolute, R, Y, u):
        R, u = R.view(-1, NP, C), u.view(-1, 4, C)[src]
        blocks = []
        for lo in range(max_ell + 1):
            js = list(per[lo])
            if "paths_swapped" in mut and lo == 1:
                js[0], js[1] = js[1], js[0]
            cols = []
            for p in js:
                li, ls, _ = paths[p]
                m = torch.einsum("eic,ej,ijk->ekc", u[:, li * li:(li + 1) ** 2], Y[:, ls * ls:(ls + 1) ** 2],
                                 cg_of(p, absolute)) * R[:, p, None, :]
                cols.append(torch.zeros(n, 2 * lo + 1, C, dtype=F64).index_add(0, dst, m))
            blk = torch.stack(cols, 2)  # [n][2lo+1][np][C] -> [2lo+1][n][np][C]
            blocks.append(blk.permute(1, 0, 2, 3).reshape(-1))
        return torch.cat(blocks)
    return f


def elem_mix_fn(c, n, C, L1, nsh, mut=()):
    """out [nsh][n][C] = in [nsh][n][C] @ W[type][l] (W [n_elem][Lw][C][C])"""
    Lw = 1 if nsh == 1 else L1
    z = c["type"][:n].long()
    if "elem_of_neighbour" in mut:
        z = z.roll(-1)
    ls = l_sel(nsh) if nsh > 1 else torch.zeros(1, dtype=torch.long)
    if "l1_block_on_l2" in mut and nsh >= 9:
        ls = ls.clone()
        ls[4:9] = 1

    def f(absolute, W, x):
        W = W.view(-1, Lw, C, C)[z]  # [n][Lw][C][C]
        return torch.einsum("knc,nkcd->knd", x.view(nsh, n, C), W[:, ls])
    return f


def elem_mix_rows_fn(c, n, C, ncomp, ldi, mut=()):
    """out rows [n][ncomp C] = in rows (pitch ldi) @ W[type][l(m)] (W [n_elem][1 or 2][C][C])"""
    Lw = 2 if ncomp == 4 else 1
    z = c["type"][:n].long()
    if "elem_of_neighbour" in mut:
        z = z.roll(-1)
    ls = torch.tensor([0, 1, 1, 1][:ncomp])

    def f(absolute, W, x):
        W = W.view(-1, Lw, C, C)[z]
        xr = x.view(n, ldi)[:, :ncomp * C].view(n, ncomp, C)
        return torch.einsum("nkc,nkcd->nkd", xr, W[:, ls]).reshape(n, ncomp * C)
    return f


# ------------------------------------------------------------------------------------------------ symmetric contraction
def make_contraction(max_ell, correlation, Cr, eq, seed):
    """the contraction module(s) of one product block (contractions.0, and .1 when eq), U and weights rounded to fp32"""
    torch.manual_seed(seed)
    n_elem = len(ELEMS)
    mods = [MR.Contraction(max_ell, correlation, n_elem, Cr)]
    if eq:
        mods.append(EQ.ContractionVec(max_ell, correlation, n_elem, Cr))
    with torch.no_grad():
        for m in mods:
            for nu in range(1, correlation + 1):
                U = getattr(m, f"U_matrix_{nu}")
                U.copy_(U.float().double())
                w = m.weight_of(nu)
                w.copy_((w * 4.0).float().double())  # weights of order one
    return mods


def stack_weights(mods, C):
    """wsym [n_elem][Ktot][C] (every nu of contractions.0, then of .1; channels padded to C) and each block's kg0"""
    blocks, kg0, k = [], [], 0
    for m in mods:
        for nu in range(1, m.correlation + 1):
            w = m.weight_of(nu).detach()
            kg0.append(k)
            k += w.shape[1]
            blocks.append(torch.nn.functional.pad(w, (0, C - w.shape[2])))
    return torch.cat(blocks, 1).float(), kg0


def build_terms(shim, mods, nsh):
    """the engine's term list (mace_sym_terms through the shim) for every U of the block, in the engine's order"""
    out, k = [], 0
    for ci, m in enumerate(mods):
        for nu in range(1, m.correlation + 1):
            U = getattr(m, f"U_matrix_{nu}").float()
            K = U.shape[-1]
            out.append(shim.mace_sym_terms(U, nsh, nu, 3 if ci else 1, K, k))
            k += K
    return torch.cat(out)


def symc_fn(mods, c, n, C, nsh, eq, mut=()):
    """B [n][C] (eq: [4][n][C], slot 0 the 0e output, 1..3 the 1o components) from A [nsh][n][C] by the contraction
    modules' own forward; `absolute`: |U|, |w|"""
    z = c["type"][:n].long()
    if "elem_of_neighbour" in mut:
        z = z.roll(-1)
    Cr = mods[0].weight_of(1).shape[2]

    def f(absolute, A):
        Ar = A.view(nsh, n, C).permute(1, 0, 2)[:, :, :Cr]
        outs = []
        for ci, m in enumerate(mods):
            mm = _mutated(m, absolute, mut, ci)
            B = mm(Ar, z)
            outs.append(B[:, None] if ci == 0 else B.permute(0, 1, 2))
        B = torch.cat(outs, 1) if eq else outs[0]  # [n][4][Cr] or [n][1][Cr]
        if eq and "o_slots_1_3_swapped" in mut:
            B = B[:, [0, 3, 2, 1]]
        B = torch.nn.functional.pad(B, (0, C - Cr))
        return B.permute(1, 0, 2).reshape(-1)
    return f


def _mutated(m, absolute, mut, ci):
    """a copy of contraction m with |U| and |w| (absolute) or a host-builder mutant applied to its U / weights"""
    mm = copy.deepcopy(m)
    with torch.no_grad():
        for nu in range(1, m.correlation + 1):
            U = getattr(mm, f"U_matrix_{nu}")
            lead = 1 if ci else 0
            if "one_permutation" in mut and nu >= 2:
                U.copy_(_one_permutation(U, nu, lead))
            if "drop_smallest_term" in mut and nu == m.correlation and ci == 0:
                U.copy_(_drop_smallest(U, nu, lead))
            if "kg_off_by_one" in mut and nu == 2 and ci == 0:
                w = mm.weight_of(nu)
                w.copy_(torch.cat([w[:, 1:], mm.weight_of(nu + 1)[:, :1] if nu < m.correlation else w[:, :1] * 0], 1))
            if absolute:
                U.abs_()
                mm.weight_of(nu).abs_()
    return mm


def _sorted_view(U, nu, lead):
    """U summed over the permutations of each sorted index tuple, as a dict of (sorted tuple) -> [(lead,) K] values"""
    import itertools
    n = U.shape[lead]
    out = {}
    for ix in itertools.combinations_with_replacement(range(n), nu):
        s = 0
        for p in set(itertools.permutations(ix)):
            s = s + (U[(slice(None),) + p] if lead else U[p])
        out[ix] = s
    return out


def _one_permutation(U, nu, lead):
    """U with each sorted tuple's entries kept at the sorted permutation only (the others zero), unsummed"""
    import itertools
    V = torch.zeros_like(U)
    n = U.shape[lead]
    for ix in itertools.combinations_with_replacement(range(n), nu):
        sl = (slice(None),) + ix if lead else ix
        V[sl] = U[sl]
    return V


def _drop_smallest(U, nu, lead):
    """U without the term (sorted tuple, k) of smallest nonzero |sum over permutations| (above the host's cut)"""
    import itertools
    sv = _sorted_view(U, nu, lead)
    umax = float(U.abs().max())
    best, key = math.inf, None
    for ix, v in sv.items():
        vv = v.reshape(-1, v.shape[-1]) if lead else v.reshape(1, -1)
        for r in range(vv.shape[0]):
            for k in range(vv.shape[1]):
                a = abs(float(vv[r, k]))
                if 1e-6 * umax < a < best:
                    best, key = a, (ix, r, k)
    V = U.clone()
    ix, r, k = key
    for p in set(itertools.permutations(ix)):
        if lead:
            V[(r,) + p + (k,)] = 0.0
        else:
            V[p + (k,)] = 0.0
    return V


def symc_terms_bwd(terms, A, w, z, gB, nsh, eq, mut=()):
    """gA [nsh][n][C] of k_mace_symc(_eq)<kBwd> walked over the term list (the reverse of a mutant kernel:
    `repeat_once` adds a repeated index's adjoint once)"""
    A = d64(A)
    n, C = A.shape[1], A.shape[2]
    w, gB = d64(w), d64(gB).view(4 if eq else 1, n, C)
    idx, kg, coef = terms[:, 0], terms[:, 1], d64(terms[:, 2].contiguous().view(torch.float32))
    gA = torch.zeros(nsh, n, C, dtype=F64)
    for j in range(len(idx)):
        t = int(idx[j])
        nu, o = (t >> 24) & 3, (t >> 28) & 3
        ii = [t & 255, (t >> 8) & 255, (t >> 16) & 255][:nu]
        s = coef[j] * w[z, int(kg[j])] * gB[o]
        a = [A[i] for i in ii]
        seen = set()
        for q in range(nu):
            if "repeat_once" in mut and ii[q] in seen:
                continue
            seen.add(ii[q])
            prod = s
            for r in range(nu):
                if r != q:
                    prod = prod * a[r]
            gA[ii[q]] += prod
    return gA


# ------------------------------------------------------------------------------------------------ readouts
def readout_final_ref(c, h, W1, w2, e_lin, E0, scale, shift, wgt, mut=()):
    """{pre [n][H], energy [1] (+ on the prefill 0), atom_e [N] (eps at gid)}; h [n][C], W1 [C][H]"""
    n = c["n_own"]
    pre = Mag(d64(h)).mm(d64(W1))
    act = silu_scale(pre.x, pre.s)
    e = act.mm(d64(w2)[:, None])[:, 0]
    z = c["type"][:n].long()
    if "e0_wrong_element" in mut:
        z = (z + 1) % len(ELEMS)
    eps = d64(E0)[z] + scale * (d64(e_lin) + e.x) + shift
    s_eps = abs(scale) * (e.s + e.x.abs() + d64(e_lin).abs()) + DBL * eps.abs()
    if wgt is not None:
        wv = d64(wgt)[c["gid"][:n].long()]
        if "wgt_twice" in mut:
            wv = wv * wv
        eps, s_eps = eps * wv, s_eps * wv.abs() + DBL * (eps * wv).abs()
    energy = Mag(eps.sum()[None], (s_eps + DBL * n * eps.abs()).sum()[None])
    return dict(pre=pre, energy=energy, eps=Mag(eps, s_eps))


def readout_seed_ref(c, pre, W1, w2, scale, wgt, mut=()):
    """gh [n][C] = scale wgt sum_j W1[c][j] w2[j] SiLU'(pre[j])"""
    n = c["n_own"]
    p = d64(pre)
    act = dsilu if "silu_p_as_sigma" not in mut else torch.sigmoid
    dp = Mag(p, 2.0 + 1.5 * p.abs()).apply(act)
    Ww = d64(W1) * d64(w2)[None, :]
    gh = dp.mm(Ww.T)
    sc = torch.full((n,), float(scale), dtype=F64)
    if wgt is not None:
        wv = d64(wgt)[c["gid"][:n].long()]
        sc = sc * (wv * wv if "wgt_twice" in mut else wv)
    return Mag(gh.x * sc[:, None], (gh.s + gh.x.abs()) * sc.abs()[:, None])


# ------------------------------------------------------------------------------------------------ edge final
def edge_energy(v, c, nb, nsh, core, g_eb, gY, wz, mut=()):
    """per-edge G(v) = g_eb . eb(|v|) + gY[1:] . Y(v) (+ zscale wgt V(|v|)) whose gradient k_mace_edge_final forms"""
    d = v.norm(dim=1)
    G = (d64(g_eb)[:, :nb] * radial_basis(d, c, nb, core, mut)[:, :nb]).sum(1)
    Y = sh(v, nsh, mut)
    gy = d64(gY).clone()
    gy[:, 0] = 0.0
    G = G + (gy[:, :nsh] * Y[:, :nsh]).sum(1)
    if "no_pr" in mut:  # the radial part of the harmonics' gradient kept: pr u / d with pr = sum_m gY_m l_m Y_m
        lm = torch.tensor(MR.l_of_index(int(round(math.sqrt(nsh))) - 1), dtype=F64)
        G = G + ((gy[:, :nsh] * lm * Y[:, :nsh]).sum(1)).detach() * torch.log(d)
    if core["zbl"]:
        G = G + wz * zbl_edge(d, c, core)
    return G


def edge_final_ref(c, nb, nsh, core, g_eb, gY, forces, virial, atom_vir, wgt, mut=()):
    """{forces [N][3], virial [9], atom_vir [N][12] (None without)}: += on the prefills"""
    v = d64(c["e_vec"][:, :3]).requires_grad_(True)
    src, dst = c["e_src"].long(), c["e_dst"].long()
    gid = c["gid"].long()
    wz = torch.full((c["E"],), core["zscale"], dtype=F64)
    if wgt is not None and core["zbl"]:
        w = d64(wgt)[gid[dst]]
        wz = wz * (w * w if "wgt_twice" in mut else w)
    f = lambda x: edge_energy(x, c, nb, nsh, core, g_eb, gY, wz, mut)  # noqa: E731
    with torch.enable_grad():
        G = f(v)
        (g,) = torch.autograd.grad(G.sum(), v, create_graph=True)
        H = [torch.autograd.grad(g[:, j].sum(), v, retain_graph=True)[0] for j in range(3)]
    g = g.detach()
    va = v.detach().abs()
    # scales: |g| + the inputs' sensitivities: sum_i |dg_j/dv_i| |v_i| and the terms of the g_eb, gY sums
    s = g.abs() + torch.stack([(H[j].abs() * va).sum(1) for j in range(3)], 1)
    vd = v.detach()
    d = vd.norm(dim=1)
    u = vd / d[:, None]
    deb = torch.func.jvp(lambda x: radial_basis(x, c, nb, core), (d,), (torch.ones_like(d),))[1][:, :nb]
    s_gd = (d64(g_eb)[:, :nb].abs() * deb.abs()).sum(1)
    bes = bessel(d, c, nb, core)
    sf, sdf = env_powf_scale(d / R_MAX, P_CUT)
    s_gd = s_gd + (d64(g_eb)[:, :nb].abs() * bes.abs()).sum(1) * sdf / R_MAX
    if core["zbl"]:
        dV = torch.func.jvp(lambda x: zbl_edge(x, c, core), (d,), (torch.ones_like(d),))[1]
        s_gd = s_gd + (wz * dV).abs()
    dY = _jvp_cols(lambda x: sh(x, nsh), vd, range(3))
    gy = d64(gY)[:, :nsh].abs().clone()
    gy[:, 0] = 0.0
    s_h = torch.stack([(gy * dY[j][:, :nsh].abs()).sum(1) for j in range(3)], 1)
    s = s + s_gd[:, None] * u.abs() + s_h * (1 + u.abs())
    out = {}
    F = d64(forces).clone()
    Fs = d64(forces).abs().clone()
    F.index_add_(0, gid[dst], -g).index_add_(0, gid[src], g)
    Fs.index_add_(0, gid[dst], s).index_add_(0, gid[src], s)
    out["forces"] = Mag(F, Fs)
    if "vir_transposed" in mut:
        ve = (g[:, :, None] * vd[:, None, :]).reshape(-1, 9)
        se = (s[:, :, None] * va[:, None, :] + g.abs()[:, :, None] * va[:, None, :]).reshape(-1, 9)
    else:
        ve = (vd[:, :, None] * g[:, None, :]).reshape(-1, 9)
        se = (va[:, :, None] * s[:, None, :] + va[:, :, None] * g.abs()[:, None, :]).reshape(-1, 9)
    out["virial"] = Mag(d64(virial) + ve.sum(0), d64(virial).abs() + se.sum(0) + DBL * ve.abs().sum(0))
    if atom_vir is not None:
        W = d64(atom_vir).clone()
        Ws = d64(atom_vir).abs().clone()
        if "atom_vir_all_dst" in mut:
            W[:, :9].index_add_(0, gid[dst], ve)
        else:
            W[:, :9].index_add_(0, gid[src], 0.5 * ve).index_add_(0, gid[dst], 0.5 * ve)
        Ws[:, :9].index_add_(0, gid[src], 0.5 * se).index_add_(0, gid[dst], 0.5 * se)
        out["atom_vir"] = Mag(W, Ws)
    return out


# ------------------------------------------------------------------------------------------------ shim front
def _a(x):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return ctypes.c_void_p(x.data_ptr())
    if isinstance(x, bool):
        return ctypes.c_int(int(x))
    if isinstance(x, int):
        return ctypes.c_int(x)
    if isinstance(x, float):
        return ctypes.c_float(x)
    return x


ST = object()  # where an entry takes the stream


def call(shim, entry, *args):
    """shim_mace_<entry>(args..., msg, msglen): tensors as pointers, int / float as c_int / c_float, ST the stream"""
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    shim._call(getattr(shim.lib, "shim_mace_" + entry), *[st if x is ST else _a(x) for x in args])


def sentinel(*shape, dev="cuda", dtype=torch.float32):
    return torch.full(shape, SENTINEL, device=dev, dtype=dtype)
