"""Kernel-unit tests of the TensorNet path: input generators and a float64 restatement of every launcher of
kernels_tn.cu with a per-element error scale, in the manner of tests/kernel_units_ref.py (whose `Mag`, `max_err`,
`check` and shim it uses) and tests/mace_units_ref.py.

The reference works on 3x3 tensors with the functions of oracle/tensornet_ref.py (`cosine_cutoff`,
`GaussianExpansion`, `vector_to_skewtensor`, `vector_to_symtensor`, `decompose_tensor`, `tensor_norm`, `torch.matmul`,
LayerNorm); the kernels' 10-row storage ([n][10][64]: I | a_x a_y a_z | S_xx S_xy S_xz S_yy S_yz S_zz, per the comment
at the top of kernels_tn.cu) is written out only in `pack` / `unpack`.  Values of every reverse launcher come from
torch.autograd of the forward restatement, never from the kernels' hand expansions (`full_adj`, `dec_adj`,
`scale_bwd10`, the `gvh` formula); `prod_bwd_hand` / `update_bwd_hand` restate two of them only to show what a
wrong one would compute (the mutants of tests/test_tn_units_cpu.py).

The stored S_zz makes the 10-row form redundant: `unpack` takes S's traceless part, so the restatement does not see
the trace direction n = (S_xx + S_yy + S_zz) of its input, and an adjoint it returns has no component along n.  The
kernels pass such a component through unchanged (`full_adj` treats S_zz as free), and every consumer of an adjoint
annihilates it (`dec_adj`, products with a traceless S, `embed_agg_bwd`'s traceless s6), so 10-row adjoints are
compared after `proj` (= pack(unpack(.))), which removes it.

Scales, in units of one fp32 rounding of the quantity they sit beside (kernel_units_ref.Mag):
  * element-wise launchers (one thread per (atom, channel)): `mapply`, the Mag rule of a vector function,
    |f| + sum_i |df/dx_i| s(x_i), stage by stage; the reverse launchers use the same rule on the vjp;
  * per-edge functions of the fp32 edge vector: |q| + sum_i |dq/dv_i| |v_i|; `__cosf` / `__sinf` add their documented
    absolute error 2^-21.41 on [-pi, pi] (else the cutoff near rc would have a zero scale);
  * SiLU, SiLU' and the gate's sigmoid through `__expf`: the argument carries 2 + 1.5 |x| (ex2.approx of x log2 e);
  * sums accumulated in double (readout energy, the virial) add 2^-29 |x| per term.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as Fn

from oracle import tensornet_ref as TR
from tests.kernel_units_ref import F64, Mag, d64

# |out - ref| <= TOL * scale, per element.  Set from the H100 run recorded in DESIGN.md section 5 (at least 3x the
# largest error observed) and at least 10x below every mutant (tests/test_tn_units_cpu.py).
TOL = {"gemm": 1.5e-6, "edge_geom": 2e-7, "embed_agg": 2e-7, "embed_agg_bwd": 2e-7, "layernorm": 3e-7,
       "layernorm_bwd": 3e-7, "node": 2.5e-6, "node_bwd": 1.5e-6, "msg": 3e-7, "msg_bwd": 5e-7, "readout": 4e-7,
       "edge_final": 2e-7}
DBL = 2.0 ** -29           # one double rounding, in units of an fp32 one
TRIG = 2.0 ** (24 - 21.41)  # __cosf / __sinf absolute error on [-pi, pi], in units of 2^-24
TC = 64
RC, WIDTH = 5.0, 0.5       # TensorNet's defaults: cutoff 5 A, Gaussian width 0.5 on [0, rc + 1]
N_ELEM = 3


def mu_of(nr):
    """the nr Gaussian centres of BondExpansion (fp32, as the engine packs them)"""
    return TR.GaussianExpansion(0.0, RC + 1.0, nr, WIDTH).centers.detach().float()


# ------------------------------------------------------------------------------------------------ storage
def unpack(t):
    """[..., 10] -> [..., 3, 3]: I eye + skew(a) + S (S's trace, zero up to rounding, dropped)"""
    sh = t.shape[:-1]
    eye = torch.eye(3, dtype=t.dtype)
    A = TR.vector_to_skewtensor(t[..., 1:4].reshape(-1, 3)).reshape(*sh, 3, 3)
    s = t[..., 4:10]
    S = torch.stack([s[..., 0], s[..., 1], s[..., 2], s[..., 1], s[..., 3], s[..., 4], s[..., 2], s[..., 4],
                     s[..., 5]], -1).reshape(*sh, 3, 3)
    S = S - (s[..., 0] + s[..., 3] + s[..., 5])[..., None, None] / 3.0 * eye
    return t[..., 0, None, None] * eye + A + S


def pack(M):
    """[..., 3, 3] -> [..., 10] by decompose_tensor"""
    I, A, S = TR.decompose_tensor(M)
    return torch.stack([I[..., 0, 0], A[..., 2, 1], A[..., 0, 2], A[..., 1, 0], S[..., 0, 0], S[..., 0, 1],
                        S[..., 0, 2], S[..., 1, 1], S[..., 1, 2], S[..., 2, 2]], -1)


def proj(t):
    """a 10-row adjoint without its component along the trace direction (module docstring)"""
    return pack(unpack(t))


def rows(t, n):
    """[n][10][64] (any float tensor) -> float64 [n * 64][10], row = atom * 64 + channel"""
    return d64(t).reshape(n, 10, TC).permute(0, 2, 1).reshape(n * TC, 10)


def lay(r, n):
    """[n * 64][k] -> [n][k][64] (a tensor or a Mag)"""
    if isinstance(r, Mag):
        return Mag(lay(r.x, n), lay(r.s, n))
    k = r.shape[-1]
    return r.reshape(n, TC, k).permute(0, 2, 1).reshape(n, k, TC)


def lay_proj(out, n):
    """device [n][10][64] adjoint -> projected [n][10][64] float64 (host)"""
    return lay(proj(rows(out.detach().cpu(), n)), n)


def mproj(m, n):
    """a [n][10][64] Mag projected: its value by proj, its scale plus |proj| of it (proj mixes the S-diagonal rows)"""
    r = mapply(proj, Mag(rows(m.x, n), rows(m.s, n)))
    return Mag(lay(r.x, n), m.s + lay(mapply(proj, Mag(torch.zeros_like(r.x), rows(m.s, n))).s, n))


# ------------------------------------------------------------------------------------------------ scale helpers
def mapply(f, *ms):
    """Mag of y = f(*x) for a row-wise f ([B][k_i] -> [B][j]): |y| + sum_i |dy/dx_i| s(x_i), by forward mode"""
    xs = tuple(m.x for m in ms)
    y = f(*xs)
    s = y.abs()
    for a, m in enumerate(ms):
        for j in range(m.x.shape[-1]):
            t = tuple(torch.zeros_like(x) for x in xs)
            t[a][..., j] = 1.0
            s = s + torch.func.jvp(f, xs, t)[1].abs() * m.s[..., j:j + 1]
    return Mag(y, s)


def vjp_of(f, nargs=1):
    """(x..., g) -> the vjp of f at x with cotangent g, concatenated over the first nargs arguments"""
    def h(*a):
        _, pull = torch.func.vjp(f, *a[:-1])
        gs = pull(a[-1])
        return torch.cat(gs[:nargs], -1)
    return h


def expf(m):
    """a Mag whose value is the argument of an __expf-based function (SiLU, SiLU', sigmoid)"""
    return Mag(m.x, m.s + 2.0 + 1.5 * m.x.abs())


def dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def dsigmoid(x):
    s = torch.sigmoid(x)
    return s * (1 - s)


# ------------------------------------------------------------------------------------------------ generators
def gen_graph(n_own, seed, counts=None, n_halo=None, empty=0, heavy=0, per_row=6, E=None):
    """One partition's CSR-by-destination graph: e_dst ascending over n_own owned atoms (`counts` edges per row if
    given, else random with `empty` rows without edges and one of `heavy` edges; E edges spread over the rows if E is
    given), e_src over n_loc = n_own + n_halo rows with a quarter of the sources in the halo, types mixed, gid a
    permutation of N = n_own + 3 global ids (halo rows images of random owned atoms, one the image of an edge's own
    destination: a self-image edge), |e_vec.xyz| = e_vec.w in fp32 with distances in [0.3, rc]: a few within 1e-4 A
    of rc and two exactly at rc."""
    g = torch.Generator().manual_seed(seed)
    n_halo = max(2, n_own // 3) if n_halo is None else n_halo
    n_loc, N = n_own + n_halo, n_own + 3
    if counts is not None:
        cnt = torch.tensor(counts, dtype=torch.long)
        assert len(cnt) == n_own
    else:
        cnt = torch.randint(1, 2 * per_row, (n_own,), generator=g)
        if n_own:
            cnt[torch.randperm(n_own, generator=g)[:empty]] = 0
            if heavy:
                cnt[int(torch.randint(0, n_own, (1,), generator=g))] = heavy
        if E is not None:
            r = torch.nonzero(cnt > 0).flatten()
            cnt = torch.bincount(r[torch.randint(0, len(r), (E,), generator=g)], minlength=n_own)
    E = int(cnt.sum())
    row_ptr = torch.cat([torch.zeros(1, dtype=torch.long), cnt.cumsum(0)]).int()
    dst = torch.repeat_interleave(torch.arange(n_own), cnt).int()
    src = torch.randint(0, n_loc, (E,), generator=g)
    if E > 3:
        sel = torch.randperm(E, generator=g)[: E // 4]
        src[sel] = torch.randint(n_own, n_loc, (len(sel),), generator=g)
    type_ = torch.randint(0, N_ELEM, (n_loc,), generator=g).int()
    gid = torch.empty(n_loc, dtype=torch.long)
    gid[:n_own] = torch.randperm(N, generator=g)[:n_own]
    gid[n_own:] = gid[:n_own][torch.randint(0, max(n_own, 1), (n_halo,), generator=g)] if n_own else 0
    if E:
        e0 = int(torch.randint(0, E, (1,), generator=g))
        h = n_own + int(torch.randint(0, n_halo, (1,), generator=g))
        src[e0] = h
        gid[h], type_[h] = gid[dst[e0].long()], type_[dst[e0].long()]
    d = 0.3 + (RC - 0.3) * torch.rand(E, generator=g, dtype=F64)
    u = torch.randn(E, 3, generator=g, dtype=F64)
    u = u / u.norm(dim=1, keepdim=True)
    if E:
        nc = torch.randperm(E, generator=g)[: max(1, E // 16)]
        d[nc] = RC - 1e-4 * torch.rand(len(nc), generator=g, dtype=F64)
    xyz = (u * d[:, None]).float()
    if E >= 8:  # exactly at rc: (3, 4, 0) rc / 5 and (0, 0, -rc) are exact in fp32, and so are their norms
        at = torch.randperm(E, generator=g)[:2]
        xyz[at[0]] = torch.tensor([3.0, 4.0, 0.0]) * (RC / 5.0)
        xyz[at[1]] = torch.tensor([0.0, 0.0, -RC])
    e_vec = torch.cat([xyz, xyz.to(F64).norm(dim=1, keepdim=True).float()], 1)
    return dict(n_own=n_own, n_loc=n_loc, N=N, E=E, row_ptr=row_ptr, e_src=src.int(), e_dst=dst, e_vec=e_vec,
                type=type_, gid=gid.int(), g=g)


def gen_dec(g, n, smin=0.03, smax=1.3):
    """[n][10][64] fp32 from random 3x3 tensors (per (atom, channel) scales log-uniform in [smin, smax], so norms
    from ~1e-2 to ~20) through decompose_tensor"""
    s = torch.exp(math.log(smin) + (math.log(smax) - math.log(smin)) * torch.rand(n, TC, 1, 1, generator=g,
                                                                                   dtype=F64))
    M = torch.randn(n, TC, 3, 3, generator=g, dtype=F64) * s
    return pack(M).float().permute(0, 2, 1).contiguous()


def rnd(g, *shape, s=1.0):
    return torch.randn(*shape, generator=g) * s


# ------------------------------------------------------------------------------------------------ row GEMM
def gemm_ref(A, B, bias=None, epi=0, Pre=None, Cold=None, accum=False, mut=()):
    """C = epi(A @ B + bias) (+ Cold if accum, after the epilogue); A [M][K], B [K][N].  Returns (C, Cpre) Mags."""
    A, B = d64(A), d64(B)
    K = A.shape[1]
    if "last_k_chunk_dropped" in mut:
        A, B = A[:, : K - 32], B[: K - 32]
    if "rows_64_127_lost" in mut:
        A = A.clone()
        A[64:128] = 0.0
    acc = Mag(A).mm(B)
    if bias is not None:
        acc = acc + Mag(d64(bias)[None, :].expand_as(acc.x))
    pre = acc
    if accum and "accum_before_dsilu" in mut:
        acc = acc + Mag(d64(Cold))
    if epi == 1:
        acc = expf(acc).apply(torch.nn.functional.silu)
    elif epi == 2:
        acc = acc * expf(Mag(d64(Pre))).apply(dsilu)
    if accum and "accum_before_dsilu" not in mut:
        acc = acc + Mag(d64(Cold))
    return acc, pre


# ------------------------------------------------------------------------------------------------ edge geometry
def edge_geom_ref(e_vec, nr, nrp=64, mut=()):
    """{rbf [E][nrp] (zero past nr), cut [E]} Mags"""
    d = d64(e_vec[:, 3])
    mu = d64(mu_of(nr))
    ge = TR.GaussianExpansion(0.0, 1.0, nr, WIDTH).double()
    with torch.no_grad():
        ge.centers.copy_(mu)
    val = ge(d).detach()
    t = Mag(d[:, None] - mu[None, :], d.abs()[:, None] + mu.abs()[None, :])
    arg = expf(Mag(-WIDTH * t.x * t.x, WIDTH * 2 * t.x.abs() * t.s))
    s = arg.apply(torch.exp).s
    E = len(d)
    rbf = Mag(torch.cat([val, torch.zeros(E, nrp - nr, dtype=F64)], 1),
              torch.cat([s, torch.zeros(E, nrp - nr, dtype=F64)], 1))
    dd = d.clone().requires_grad_(True)
    with torch.enable_grad():
        c = TR.cosine_cutoff(dd, RC)
        (dc,) = torch.autograd.grad(c.sum(), dd)
    inside = (d <= RC).to(F64)
    cut = Mag(c.detach(), c.detach().abs() + 3.0 * dc.abs() * d + 0.5 * TRIG * inside)
    return dict(rbf=rbf, cut=cut)


# ------------------------------------------------------------------------------------------------ embedding
def _unit(e_vec):
    """v^ = xyz / w from the fp32 edge vector (the kernels divide by e_vec.w) and its Mag"""
    ev = Mag(d64(e_vec))
    return mapply(lambda v: v[:, :3] / v[:, 3:4], ev)


def _dirs(vn):
    """[E][3][10]: pack(eye), pack(skew(v^)), pack(sym(v^)) -- the three edge tensors of TensorEmbedding"""
    eye = torch.eye(3, dtype=vn.dtype).expand(len(vn), 3, 3)
    return torch.stack([pack(eye), pack(TR.vector_to_skewtensor(vn)), pack(TR.vector_to_symtensor(vn))], 1)


def _zij(c, U, V, mut=()):
    src, dst, ty = c["e_src"].long(), c["e_dst"].long(), c["type"].long()
    if "uv_swapped" in mut:
        src, dst = dst, src
    return U[ty[src]] + V[ty[dst]]


def embed_agg_values(c, U, V, P, cut, vn, mut=()):
    """T [n_own][64][3][3] of TensorEmbedding's aggregation (plain float64, autograd-able); P [E][3][64]"""
    dst = c["e_dst"].long()
    Cz = cut[:, None] * _zij(c, U, V, mut)  # [E][64]
    eye = torch.eye(3, dtype=F64)
    Iij = (P[:, 0] * Cz)[..., None, None] * eye
    Aij = (P[:, 1] * Cz)[..., None, None] * TR.vector_to_skewtensor(vn)[:, None]
    Sij = (P[:, 2] * Cz)[..., None, None] * TR.vector_to_symtensor(vn)[:, None]
    return torch.zeros(c["n_own"], TC, 3, 3, dtype=F64).index_add(0, dst, Iij + Aij + Sij)


def embed_agg_ref(c, U, V, P, cut, gT0=None, gC0=None, mut=()):
    """forward {T0 [n][10][64], nr0 [n][64]} and, with gT0 ([n][10][64]) and the gC prefill, the reverse
    {gP [E][192], gC [E], gvh [E][3]}: values by the 3x3 restatement and autograd, scales by Mags on the 10 rows"""
    n, E = c["n_own"], c["E"]
    src, dst, ty = c["e_src"].long(), c["e_dst"].long(), c["type"].long()
    U, V, P, cut = d64(U), d64(V), d64(P).reshape(E, 3, TC), d64(cut)
    vn_m = _unit(c["e_vec"])
    vn = vn_m.x.clone().requires_grad_(True)
    Pl, cl = P.clone().requires_grad_(True), cut.clone().requires_grad_(True)
    with torch.enable_grad():
        T = embed_agg_values(c, U, V, Pl, cl, vn, mut)
        T0 = pack(T)
        if "no_traceless" in mut:  # sym(v^) without its -|v^|^2/3 on the diagonal: S_xx, S_yy, S_zz rows + w3 |v^|^2/3
            q = torch.zeros(n, TC, dtype=F64).index_add(
                0, c["e_dst"].long(), Pl[:, 2] * (cl[:, None] * _zij(c, U, V)) * ((vn * vn).sum(1) / 3.0)[:, None])
            z = torch.zeros_like(q)
            T0 = T0 + torch.stack([z, z, z, z, q, z, z, q, z, q], -1)
        out = {}
        if gT0 is not None:
            gt = d64(gT0).reshape(n, 10, TC).permute(0, 2, 1)
            gP, gCv, gv = torch.autograd.grad((T0 * gt).sum(), [Pl, cl, vn], allow_unused=True)
    T0, T = T0.detach(), T.detach()
    # scales on the 10 rows: contribution_e = sum_p P_p C Z D_p(v^)
    Dm = mapply(lambda v: _dirs(v).reshape(len(v), 30), vn_m)
    Dm = Mag(Dm.x.reshape(E, 3, 10), Dm.s.reshape(E, 3, 10))
    Zm = Mag(U)[ty[src]] + Mag(V)[ty[dst]]
    Cz = Mag(cut)[:, None] * Zm  # [E][64]
    wp = [Mag(P[:, p]) * Cz for p in range(3)]
    terms = [wp[p][:, :, None] * Dm[:, p][:, None, :] for p in range(3)]
    contrib = terms[0] + terms[1] + terms[2]
    s_T0 = torch.zeros(n, TC, 10, dtype=F64).index_add(0, dst, contrib.s)
    T0m = Mag(T0, s_T0)
    nr0 = mapply(lambda t: TR.tensor_norm(unpack(t))[:, None], Mag(T0.reshape(-1, 10), s_T0.reshape(-1, 10)))
    nr0 = Mag(TR.tensor_norm(T).reshape(-1, 1), nr0.s)
    out.update(T0=Mag(T0.permute(0, 2, 1), T0m.s.permute(0, 2, 1)), nr0=Mag(nr0.x.reshape(n, TC), nr0.s.reshape(n, TC)))
    if gT0 is None:
        return out
    g10 = Mag(d64(gT0).reshape(n, 10, TC).permute(0, 2, 1))[dst]  # [E][64][10]
    gw = [(g10 * Dm[:, p][:, None, :]).sum(2) for p in range(3)]  # [E][64]
    gPm = [gw[p] * Cz for p in range(3)]
    gPs = torch.stack([m.s for m in gPm], 1).reshape(E, 3 * TC)
    out["gP"] = Mag(gP.reshape(E, 3 * TC), gPs)
    rc = sum((gw[p] * Mag(P[:, p]) * Zm for p in range(1, 3)), gw[0] * Mag(P[:, 0]) * Zm).sum(1)
    out["gC"] = Mag(d64(gC0) + gCv, d64(gC0).abs() + rc.s)
    gD = [(g10 * wp[p][:, :, None]).sum(1) for p in range(3)]  # [E][10]
    gDm = Mag(torch.stack([m.x for m in gD], 1).reshape(E, 30), torch.stack([m.s for m in gD], 1).reshape(E, 30))
    gvm = mapply(vjp_of(lambda v: _dirs(v).reshape(len(v), 30)), vn_m, gDm)
    out["gvh"] = Mag(gv, gvm.s)
    return out


# ------------------------------------------------------------------------------------------------ LayerNorm
def layernorm_ref(x, gamma, beta, gy=None, mut=()):
    """{y, stats [rows][2] (mean, rstd)} and with gy {gx}"""
    x, gamma, beta = d64(x), d64(gamma), d64(beta)
    W = x.shape[1]

    def f(xx):
        return Fn.layer_norm(xx, (W,), gamma, beta, eps=1e-5)

    xm = Mag(x)
    y = mapply(f, xm)
    xh = (x - x.mean(1, keepdim=True)) / torch.sqrt(x.var(1, unbiased=False, keepdim=True) + 1e-5)
    out = dict(y=Mag(y.x, y.s + (xh * gamma).abs() + beta.abs()))
    mean = mapply(lambda xx: xx.mean(1, keepdim=True), xm)
    rstd = mapply(lambda xx: 1.0 / torch.sqrt(xx.var(1, unbiased=False, keepdim=True) + 1e-5), xm)
    out["stats"] = Mag(torch.cat([mean.x, rstd.x], 1), torch.cat([mean.s, rstd.s], 1))
    if gy is None:
        return out

    def fb(xx, g):
        if "no_xhat_term" in mut:
            r = 1.0 / torch.sqrt(xx.var(1, unbiased=False, keepdim=True) + 1e-5)
            gh = g * gamma
            return r * (gh - gh.mean(1, keepdim=True))
        return vjp_of(f)(xx, g)
    out["gx"] = mapply(fb, xm, Mag(d64(gy)))
    return out


# ------------------------------------------------------------------------------------------------ element-wise node ops
def norm_mut(M):
    """tensor_norm with weight 1 instead of 2 on S's off-diagonal pairs (a mutant's norm)"""
    I, A, S = TR.decompose_tensor(M)
    d = torch.diagonal(S, dim1=-2, dim2=-1)
    return TR.tensor_norm(I) + TR.tensor_norm(A) + 0.5 * (TR.tensor_norm(S) + (d * d).sum(-1))


def scale_f(x, mut=()):
    M = unpack(x)
    q = TR.tensor_norm(M) + 1
    if "nw_offdiag_1" in mut:  # the norm's weights wrong in the reverse only (the forward's q is read)
        nm = norm_mut(M)
        q = q.detach() + nm - nm.detach()
    return pack(M / q[..., None, None])


def q_f(x):
    return (TR.tensor_norm(unpack(x)) + 1)[..., None]


def invariants_f(x, mut=()):
    I, A, S = TR.decompose_tensor(unpack(x))
    nS = TR.tensor_norm(S)
    if "nw_offdiag_1" in mut:
        d = torch.diagonal(S, dim1=-2, dim2=-1)
        nS = 0.5 * (nS + (d * d).sum(-1))
    return torch.stack([TR.tensor_norm(I), TR.tensor_norm(A), nS], -1)


def product_f(m, y, so3, mut=()):
    """TensorNetInteraction's product, decompose(msg Y + Y msg) (O(3)) or decompose(2 Y msg) (SO(3)), over norm + 1"""
    Mm, Y = unpack(m), unpack(y)
    if so3:
        P = 2 * torch.matmul(Mm, Y) if "so3_order_swapped" in mut else 2 * torch.matmul(Y, Mm)
    else:
        P = torch.matmul(Mm, Y) + torch.matmul(Y, Mm)
    I, A, S = TR.decompose_tensor(P)
    normp1 = (TR.tensor_norm(I + A + S) + 1)[..., None, None]
    return pack((I + A + S) / normp1)


def update_f(xh, d):
    X, dX = unpack(xh), unpack(d)
    return pack(X + dX + torch.matmul(dX, dX))


def embed_out_f(t, s):
    """X0 of TensorEmbedding from T0m rows t [B][10] and the three scalars s [B][3] (pre-activation)"""
    I, A, S = TR.decompose_tensor(unpack(t))
    a = torch.nn.functional.silu(s)
    return pack(I * a[:, 0, None, None] + A * a[:, 1, None, None] + S * a[:, 2, None, None])


def node_ref(op, n, ins, g=None, so3=0, mut=()):
    """Forward (g None) or reverse of an element-wise launcher on [n][..][64] inputs, as Mags laid out like the
    kernel's outputs.  op: "scale" ({Xh, q}), "prod" ({Pn}), "update" ({Xn}), "invariants" ({inv}), "embed_out"
    ({X0}), "norm" (nr0 of T0: the reverse only, {gT0}); reverse: {gX} / {gmsg, gY} / {gdX} / {gX} / {gT0m, gs2p}."""
    R = lambda t: Mag(rows(t, n))  # noqa: E731
    if op == "scale":
        f, a = (lambda x: scale_f(x, mut)), [R(ins[0])]
    elif op == "prod":
        f, a = (lambda m, y: product_f(m, y, so3, mut)), [R(ins[0]), R(ins[1])]
    elif op == "update":
        f, a = update_f, [R(ins[0]), R(ins[1])]
    elif op == "invariants":
        f, a = (lambda x: invariants_f(x, mut)), [R(ins[0])]
    elif op == "embed_out":
        s2p = d64(ins[1]).reshape(n, TC, 3)
        if "s2p_blocked" in mut:
            s2p = d64(ins[1]).reshape(n, 3, TC).permute(0, 2, 1)
        f, a = embed_out_f, [R(ins[0]), expf(Mag(s2p.reshape(n * TC, 3)))]
    elif op == "norm":
        f, a = (lambda x: TR.tensor_norm(unpack(x))[..., None]), [R(ins[0])]
    if g is None:
        if op == "scale":
            q = mapply(q_f, *a)
            return dict(Xh=lay(mapply(f, *a), n), q=Mag(q.x.reshape(n, TC), q.s.reshape(n, TC)))
        if op == "invariants":
            m = mapply(f, *a)  # [n*64][3] -> blocked [n][3][64]
            return dict(inv=Mag(m.x.reshape(n, TC, 3).permute(0, 2, 1), m.s.reshape(n, TC, 3).permute(0, 2, 1)))
        return {dict(prod="Pn", update="Xn", embed_out="X0")[op]: lay(mapply(f, *a), n)}
    if op == "invariants":
        gm = Mag(d64(g).reshape(n, 3, TC).permute(0, 2, 1).reshape(n * TC, 3))
    elif op == "norm":
        gm = Mag(d64(g).reshape(n * TC, 1))
    else:
        gm = R(g)
    if op == "update":  # the adjoint of dX only (the caller reuses gXn as the adjoint of Xh)
        m = mapply(vjp_of(lambda d, xh: f(xh, d)), a[1], a[0], gm)
        return dict(gdX=lay(m, n))
    nargs = 2 if op in ("prod", "embed_out") else 1
    m = mapply(vjp_of(f, nargs), *a, gm)
    if op == "prod":
        return dict(gmsg=lay(m[:, :10], n), gY=lay(m[:, 10:], n))
    if op == "embed_out":
        gs = m[:, 10:]
        return dict(gT0m=lay(m[:, :10], n), gs2p=Mag(gs.x.reshape(n, 3 * TC), gs.s.reshape(n, 3 * TC)))
    return {dict(scale="gX", invariants="gX", norm="gT0")[op]: lay(m, n)}


# ------------------------------------------------------------------------------------------------ message
def msg_contrib(f3, cut, y, mut=()):
    """one edge's message to its destination, per channel: sum_p silu(f3p_p) C part_p(Y[src]) -- [B][10];
    f3 [B][3] pre-activations (interleaved 3c + p), cut [B][1], y [B][10]"""
    I, A, S = TR.decompose_tensor(unpack(y))
    fe = torch.nn.functional.silu(f3) * cut
    return pack(I * fe[:, 0, None, None] + A * fe[:, 1, None, None] + S * fe[:, 2, None, None])


def msg_ref(c, f3p, cut, Y, gmsg=None, gC0=None, gY0=None, mut=()):
    """forward {msg [n_own][10][64]}; with gmsg and the prefills the reverse {g3 [E][192], gC [E], gY [n_loc][10][64]
    (+= on gY0, projected)}"""
    n, E, nl = c["n_own"], c["E"], c["n_loc"]
    src, dst = c["e_src"].long(), c["e_dst"].long()
    f3 = d64(f3p).reshape(E, TC, 3)
    if "f3p_blocked" in mut:
        f3 = d64(f3p).reshape(E, 3, TC).permute(0, 2, 1)
    f3 = expf(Mag(f3.reshape(E * TC, 3)))
    cm = Mag(d64(cut)[:, None].expand(E, TC).reshape(E * TC, 1))
    ym = Mag(rows(Y, nl).reshape(nl, TC, 10)[src].reshape(E * TC, 10))
    if gmsg is None:
        m = mapply(msg_contrib, f3, cm, ym)
        x = torch.zeros(n, TC, 10, dtype=F64).index_add(0, dst, m.x.reshape(E, TC, 10))
        s = torch.zeros(n, TC, 10, dtype=F64).index_add(0, dst, m.s.reshape(E, TC, 10))
        return dict(msg=Mag(x.permute(0, 2, 1), s.permute(0, 2, 1)))
    gm = Mag(rows(gmsg, n).reshape(n, TC, 10)[dst].reshape(E * TC, 10))
    m = mapply(vjp_of(msg_contrib, 3), f3, cm, ym, gm)  # [E*64][3 + 1 + 10]
    g3 = m[:, :3]
    gC = m[:, 3].x.reshape(E, TC).sum(1), m[:, 3].s.reshape(E, TC).sum(1)
    to = dst if "gy_to_dst" in mut else src
    gy0 = mproj(Mag(d64(gY0)), nl)
    gy0 = Mag(gy0.x.permute(0, 2, 1), gy0.s.permute(0, 2, 1))
    gyx = gy0.x.clone().index_add_(0, to, m.x[:, 4:].reshape(E, TC, 10))
    gys = gy0.s.clone().index_add_(0, to, m.s[:, 4:].reshape(E, TC, 10))
    return dict(g3=Mag(g3.x.reshape(E, 3 * TC), g3.s.reshape(E, 3 * TC)),
                gC=Mag(d64(gC0) + gC[0], d64(gC0).abs() + gC[1]),
                gY=Mag(gyx.permute(0, 2, 1), gys.permute(0, 2, 1)))


# ------------------------------------------------------------------------------------------------ readout
def readout_final_ref(c, n, W, hL, wL, bL, hG, wG, bG, eref, scale, mean, wgt, energy0, mut=()):
    """GatedMLP's last layer (layers: linear; gates: sigmoid) and potential_ref's scaling, per owned row:
    {lout, gout, e_atom, energy [1] (+= energy0), atom_e [n] (at gid)}"""
    L = Mag(d64(hL)).mm(d64(wL)[:, None])[:, 0] + Mag(torch.full((n,), float(bL), dtype=F64))
    b = Mag(d64(hG)).mm(d64(wG)[:, None])[:, 0] + Mag(torch.full((n,), float(bG), dtype=F64))
    G = expf(b).apply(torch.sigmoid)
    e = L * G
    ev = Mag(float(scale) * e.x, abs(float(scale)) * e.s + DBL * (float(scale) * e.x).abs())
    ty = c["type"][:n].long()
    if eref is not None:
        if "eref_wrong_element" in mut:
            ty = (ty + 1) % N_ELEM
        r = d64(eref)[ty]
        ev = Mag(ev.x + r, ev.s + DBL * (ev.x + r).abs())
    mpa = torch.full((n,), float(mean), dtype=F64)
    if wgt is not None:
        w = d64(wgt)[c["gid"][:n].long()]
        if "wgt_twice" in mut:
            w = w * w
        ev = Mag(ev.x * w, ev.s * w.abs() + DBL * (ev.x * w).abs())
        mpa = mpa * w
    ae = Mag(ev.x + mpa, ev.s + DBL * (ev.x + mpa).abs() + DBL * mpa.abs())
    e0 = d64(energy0)
    tot = Mag(e0 + ev.x.sum(), e0.abs() + ev.s.sum() + DBL * n * ev.x.abs().sum())
    return dict(lout=L, gout=G, e_atom=Mag(e.x, e.s + e.x.abs()), energy=tot, atom_e=ae)


def readout_seed_ref(c, n, lout, gout, scale, wL, wG, preL, preG, wgt):
    """{gL, gG} [n][W]: adjoints of the last hidden pre-activations of both chains of E = sum scale wgt L G, with
    L = silu(preL) wL + b_L and G = sigmoid(silu(preG) wG + b_G), b_L / b_G per row so that L = lout and G = gout"""
    pL, pG = d64(preL).clone().requires_grad_(True), d64(preG).clone().requires_grad_(True)
    wLd, wGd = d64(wL), d64(wG)
    sc = readout_seed_scale(c, n, scale, wgt)
    Lv, Gv = d64(lout), d64(gout)
    with torch.enable_grad():
        hl = torch.nn.functional.silu(pL) @ wLd
        hg = torch.nn.functional.silu(pG) @ wGd
        L = hl + (Lv - hl).detach()
        G = torch.sigmoid(hg + (torch.special.logit(Gv) - hg).detach())
        gl, gg = torch.autograd.grad((sc * L * G).sum(), [pL, pG])
    scm = sc.abs()[:, None]
    dL = expf(Mag(d64(preL))).apply(dsilu)
    dG = expf(Mag(d64(preG))).apply(dsilu)
    Gm, Lm = Mag(Gv[:, None]), Mag(Lv[:, None])
    sL = (Gm * Mag(wLd[None, :]) * dL).s * scm + gl.abs()
    g1 = Mag(1 - Gv[:, None], Gv[:, None].abs() + (1 - Gv[:, None]).abs())
    sG = (Lm * Gm * g1 * Mag(wGd[None, :]) * dG).s * scm + gg.abs()
    return dict(gL=Mag(gl, sL), gG=Mag(gg, sG))


def readout_seed_scale(c, n, scale, wgt, mut=()):
    sc = torch.full((n,), float(scale), dtype=F64)
    if wgt is not None:
        w = d64(wgt)[c["gid"][:n].long()]
        sc = sc * (w * w if "wgt_twice" in mut else w)
    return sc


def readout_seed_mutant(c, n, lout, gout, scale, wL, wG, preL, preG, wgt, mut):
    """what k_tn_readout_seed computes with one factor wrong: "silu_p_as_sigma" (sigma' for SiLU'), "no_g1mg" (G(1-G)
    dropped), "wgt_twice" -- {gL, gG} values"""
    sc = readout_seed_scale(c, n, scale, wgt, mut)[:, None]
    act = dsigmoid if "silu_p_as_sigma" in mut else dsilu
    L, G = d64(lout)[:, None], d64(gout)[:, None]
    gate = torch.ones_like(G) if "no_g1mg" in mut else G * (1 - G)
    return dict(gL=sc * G * d64(wL)[None, :] * act(d64(preL)), gG=sc * L * gate * d64(wG)[None, :] * act(d64(preG)))


# ------------------------------------------------------------------------------------------------ edge final
def edge_energy(v, nr, g_rbf, gC, gvh, mut=()):
    """per-edge G(v) = g_rbf . rbf(|v|) + gC cut(|v|) + gvh . v / |v|, whose gradient k_tn_edge_final forms"""
    d = v.norm(dim=1)
    mu = d64(mu_of(nr))
    t = d[:, None] - mu[None, :]
    rb = torch.exp(-WIDTH * t * t)
    if "gauss_no_2" in mut:  # d rbf / dd with -w t instead of -2 w t
        rb = rb.detach() + 0.5 * (rb - rb.detach())
    C = TR.cosine_cutoff(d, RC)
    if "cut_sign" in mut:
        C = C.detach() - (C - C.detach())
    G = (d64(g_rbf)[:, :nr] * rb).sum(1) + d64(gC) * C
    u = v / d[:, None]
    if "no_tangential" in mut:  # gvh / d kept, its radial part (gvh . u) u / d not removed
        u = v / d.detach()[:, None]
    return G + (d64(gvh) * u).sum(1)


def edge_final_ref(c, nr, g_rbf, gC, gvh, forces, virial, atom_vir, mut=()):
    """{gd [E] (=), forces [N][3], virial [9], atom_vir [N][12] (None without)}: += on the prefills"""
    v = d64(c["e_vec"][:, :3]).requires_grad_(True)
    src, dst, gid = c["e_src"].long(), c["e_dst"].long(), c["gid"].long()
    E = c["E"]
    f = lambda x: edge_energy(x, nr, g_rbf, gC, gvh, mut)  # noqa: E731
    with torch.enable_grad():
        G = f(v)
        (g,) = torch.autograd.grad(G.sum(), v, create_graph=True)
        H = [torch.autograd.grad(g[:, j].sum(), v, retain_graph=True)[0] for j in range(3)]
    g = g.detach()
    vd, va = v.detach(), v.detach().abs()
    d = vd.norm(dim=1)
    u = vd / d[:, None]
    mu = d64(mu_of(nr))
    dr = d.clone().requires_grad_(True)
    with torch.enable_grad():
        t = dr[:, None] - mu[None, :]
        rb = torch.exp(-WIDTH * t * t)
        C = TR.cosine_cutoff(dr, RC)
        if "cut_sign" in mut:
            C = C.detach() - (C - C.detach())
        if "gauss_no_2" in mut:
            rb = rb.detach() + (rb - rb.detach()) * 0.5
        (drb,) = torch.autograd.grad(rb, dr, torch.ones_like(rb) * d64(g_rbf)[:, :nr], create_graph=True)
        (dC,) = torch.autograd.grad(C.sum(), dr, create_graph=True)
        gd = drb + d64(gC) * dC
        (gdd,) = torch.autograd.grad(gd.sum(), dr)
    gd = gd.detach()
    t = t.detach()
    arg = WIDTH * t * t
    rbp = (torch.exp(-arg) * 2 * WIDTH * t).abs()
    inside = (d <= RC).to(F64)
    s_gd = (d64(g_rbf)[:, :nr].abs() * rbp * (3.0 + 1.5 * arg + 2 * arg)).sum(1) + \
        d64(gC).abs() * (dC.detach().abs() + 0.5 * math.pi / RC * TRIG * inside)
    s_h = d64(gvh).abs().sum(1, keepdim=True) / d[:, None]
    s = g.abs() + torch.stack([(H[j].abs() * va).sum(1) for j in range(3)], 1) + s_gd[:, None] * u.abs() \
        + s_h * (1 + u.abs())
    out = dict(gd=Mag(gd, gd.abs() + s_gd + gdd.abs() * d))
    F = d64(forces).clone().index_add_(0, gid[dst], -g).index_add_(0, gid[src], g)
    Fs = d64(forces).abs().clone().index_add_(0, gid[dst], s).index_add_(0, gid[src], s)
    out["forces"] = Mag(F, Fs)
    if "vir_transposed" in mut:
        ve = (g[:, :, None] * vd[:, None, :]).reshape(-1, 9)
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


# ------------------------------------------------------------------------------------------------ hand reverses
def prod_bwd_hand(m, y, gPn, so3, mut=()):
    """the reverse k_tn_prod_bwd forms by hand, on rows [B][10] (float64): G = dec_adj(scale_bwd(gPn)), gM, gY in 3x3,
    back through full_adj; mut: "gm_y_not_yt" (O(3) gM = G Y + Y^T G), "dec_adj_no_trace" (dec_adj's trace term
    dropped).  Without mut it equals autograd (tests/test_tn_units_cpu.py)."""
    Mm, Y = unpack(m), unpack(y)
    P = 2 * torch.matmul(Y, Mm) if so3 else torch.matmul(Mm, Y) + torch.matmul(Y, Mm)
    pd = pack(P)
    _, pull = torch.func.vjp(lambda p: p / (TR.tensor_norm(unpack(p)) + 1)[..., None], pd)
    (gpd,) = pull(gPn)
    _, pull = torch.func.vjp(pack, P)
    (G,) = pull(gpd)
    if "dec_adj_no_trace" in mut:  # dec_adj's t = (g_I - g_Sxx - g_Syy - g_Szz) / 3 on the diagonal dropped
        t = (gpd[:, 0] - gpd[:, 4] - gpd[:, 7] - gpd[:, 9]) / 3.0
        G = G - t[:, None, None] * torch.eye(3, dtype=F64)
    Yt, Mt = Y.transpose(-2, -1), Mm.transpose(-2, -1)
    if so3:
        gM, gY = 2 * torch.matmul(Yt, G), 2 * torch.matmul(G, Mt)
    else:
        gM = (torch.matmul(G, Y) if "gm_y_not_yt" in mut else torch.matmul(G, Yt)) + torch.matmul(Yt, G)
        gY = torch.matmul(Mt, G) + torch.matmul(G, Mt)
    _, pm = torch.func.vjp(unpack, m)
    _, py = torch.func.vjp(unpack, y)
    return proj(pm(gM)[0]), proj(py(gY)[0])


def update_bwd_hand(d, g, mut=()):
    """gdX = gXn + full_adj(G D^T + D^T G), G = dec_adj(gXn); mut "d_not_dt": G D + D^T G"""
    D = unpack(d)
    _, pull = torch.func.vjp(pack, D)
    (G,) = pull(g)
    Dt = D.transpose(-2, -1)
    T = (torch.matmul(G, D) if "d_not_dt" in mut else torch.matmul(G, Dt)) + torch.matmul(Dt, G)
    _, pu = torch.func.vjp(unpack, d)
    return proj(g + pu(T)[0])
