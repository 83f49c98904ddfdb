"""Each TensorNet launcher of kernels_tn.cu on its own, called through tests/kernel_shim.cu on synthetic inputs that
meet the engine's contract (tests/tn_units_ref.py), against a float64 restatement in the 3x3 form of
oracle/tensornet_ref.py.

Every element must satisfy |out - ref| <= tol * scale (the first-order rounding bound of tn_units_ref.py); where a
kernel zero-fills (rbf padding columns, atoms without edges) the scale is 0 and the output must be exactly 0; rows,
columns and planes a launch must not write keep their sentinels or prefills bit for bit.  10-row adjoints are compared
without their component along the trace direction, which no consumer reads (tn_units_ref.py).  The cases aim at
partial last blocks, n_own * 64 % 256 != 0, n_own = 0 and E = 0, atoms without edges, a row of 300 edges, halo
sources, a self-image edge, distances at and within 1e-4 A of the cutoff, NaN in g_rbf's padding columns, runs of
equal destinations across the 32-lane and 256-thread boundaries, every row-GEMM shape the engine issues, and every
instantiation of the readout and final kernels.

B2M_TN_UNITS_REPORT=<path> writes the largest normalised error of every launcher output to <path> (JSON).
"""
import json
import os

import pytest
import torch

from tests import kernel_units_ref as KU
from tests import tn_units_ref as T

pytestmark = pytest.mark.gpu
ERRS = {}
SENT = KU.SENTINEL


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = KU.Shim(KU.build_shim(tmp_path_factory.mktemp("kernel_shim")))
    yield s
    path = os.environ.get("B2M_TN_UNITS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({k: ERRS[k] for k in sorted(ERRS)}, f, indent=1)
    for k in sorted(ERRS):
        print(f"tn-units max |out - ref| / scale  {k:<26s} {ERRS[k]:.3e}")


def check(key, tol, out, ref, what=""):
    KU.check(ERRS, key, T.TOL[tol], out, ref, what)


def check_adj(key, tol, out, ref, n, what=""):
    """a [n][10][64] adjoint, projected (tn_units_ref.proj; the kernel's rounding of each row carried through it)"""
    KU.check(ERRS, key, T.TOL[tol], T.lay_proj(out, n), T.mproj(KU.Mag(ref.x, ref.s), n), what)


def same(name, out, before, what=""):
    """out equals before bit for bit"""
    o, b = out.detach().cpu().contiguous(), before.detach().cpu().contiguous()
    v = torch.int32 if o.dtype == torch.float32 else torch.int64
    assert torch.equal(o.view(-1).view(v), b.view(-1).view(v)), f"{name} {what} changed"


def sentinel(*shape, dtype=torch.float32):
    return torch.full(shape, SENT, device="cuda", dtype=dtype)


def dev(c):
    return {k: v.cuda() for k, v in c.items() if isinstance(v, torch.Tensor)}


def sync():
    torch.cuda.synchronize()


def std_graph(seed):
    """atoms without edges, a 300-edge row, halo sources, a self-image edge; n_own * 64 % 256 != 0"""
    return T.gen_graph(37, seed, empty=3, heavy=300)


# ------------------------------------------------------------------------------------------------ row GEMM
# (K, N, epi, bias, accum): every shape and epilogue the engine issues (engine_tn.inl), readout widths 64 and 128, and
# epi 2 / epi 1 with accum (the documented order: the old C is added after the epilogue)
GEMMS = [(64, 128, 1, True, False), (128, 192, 0, True, False), (192, 64, 0, True, False), (64, 192, 0, False, False),
         (192, 128, 2, False, False), (128, 64, 0, False, False), (64, 64, 1, True, False), (128, 128, 1, True, False),
         (128, 128, 2, False, False), (64, 64, 2, False, False), (128, 64, 0, False, True), (64, 64, 0, False, True),
         (192, 128, 2, False, True), (64, 128, 1, True, True)]


@pytest.mark.parametrize("M", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("K,N,epi,bias,accum", GEMMS, ids=[f"{k}x{n}_e{e}{'_b' if b else ''}{'_acc' if a else ''}"
                                                           for k, n, e, b, a in GEMMS])
def test_gemm(shim, K, N, epi, bias, accum, M):
    g = torch.Generator().manual_seed(K + 7 * N + 31 * epi + M + 3 * accum)
    lda, ldc, ldp = K + 32, N + 64, N + 64  # strided operands: sentinels in the columns past N and rows past M
    A = torch.full((M + 3, lda), float("nan"))
    A[:M, :K] = T.rnd(g, M, K)
    B = T.rnd(g, K, N, s=K ** -0.5)
    b = T.rnd(g, N) if bias else None
    Pre = T.rnd(g, M, ldp, s=2.0)
    C0 = torch.full((M + 3, ldc), SENT)
    C0[:M, :N] = T.rnd(g, M, N)
    C = C0.cuda()
    Cpre = sentinel(M + 3, ldc) if epi == 1 else None
    shim.tn_gemm(A.cuda(), lda, B.cuda(), C, ldc, M, N, K, bias=None if b is None else b.cuda(), epi=epi,
                 Cpre=Cpre, Pre=Pre.cuda() if epi == 2 else None, ldp=ldp, accum=accum)
    sync()
    ref, pre = T.gemm_ref(A[:M, :K], B, b, epi, Pre[:M, :N], C0[:M, :N], accum)
    what = f"K={K} N={N} epi={epi} M={M}"
    check("tn_gemm C", "gemm", C[:M, :N], ref, what)
    same("C columns past N / rows past M", torch.cat([C[:, N:].reshape(-1), C[M:].reshape(-1)]),
         torch.cat([C0[:, N:].reshape(-1), C0[M:].reshape(-1)]), what)
    if epi == 1:
        check("tn_gemm Cpre", "gemm", Cpre[:M, :N], pre, what)
        assert bool((Cpre[:, N:] == SENT).all() and (Cpre[M:] == SENT).all()), f"Cpre written outside {what}"


@pytest.mark.parametrize("accum", [False, True], ids=["set", "accum"])
@pytest.mark.parametrize("M", [1, 129, 300])
def test_gemm_mix(shim, M, accum):
    """the channel mix: ten z planes of [M][64] at pitch 640, B0 for plane 0, B1 for 1..3, B2 for 4..9"""
    g = torch.Generator().manual_seed(900 + M + accum)
    X = T.gen_dec(g, M).reshape(M, 640)
    Bs = [T.rnd(g, 64, 64, s=0.125) for _ in range(3)]
    C0 = torch.cat([T.gen_dec(g, M).reshape(M, 640), torch.full((2, 640), SENT)])
    C = C0.cuda()
    shim.tn_gemm(X.cuda(), 640, Bs[0].cuda(), C, 640, M, 64, 64, zA=64, B1=Bs[1].cuda(), B2=Bs[2].cuda(), bsel=True,
                 zC=64, accum=accum, nz=10)
    sync()
    for z in range(10):
        B = Bs[0 if z == 0 else (1 if z < 4 else 2)]
        ref, _ = T.gemm_ref(X[:, 64 * z:64 * z + 64], B, Cold=C0[:M, 64 * z:64 * z + 64], accum=accum)
        check("tn_gemm mix", "gemm", C[:M, 64 * z:64 * z + 64], ref, f"M={M} z={z}")
    same("mix rows past M", C[M:], C0[M:])


def test_gemm_refusals(shim):
    """shapes the kernel cannot run are refused on the host, before any launch"""
    A, B, C = sentinel(4, 256), sentinel(256, 256), sentinel(4, 256)
    P = sentinel(4, 256)
    bad = [dict(K=48, N=64), dict(K=64, N=96), dict(K=64, N=64, epi=1, Cpre=P, nz=10),
           dict(K=64, N=64, epi=2, Pre=P, ldp=256, nz=10), dict(K=64, N=64, epi=1)]
    for kw in bad:
        K, N = kw.pop("K"), kw.pop("N")
        with pytest.raises(RuntimeError, match="b2m error"):
            shim.tn_gemm(A, 256, B, C, 256, 4, N, K, **kw)
    sync()
    assert bool((C == SENT).all() and (P == SENT).all())


# ------------------------------------------------------------------------------------------------ edge geometry
@pytest.mark.parametrize("nr", [1, 20, 64])
def test_edge_geom(shim, nr):
    for c in (std_graph(40 + nr), T.gen_graph(5, 41 + nr, E=257)):
        E = c["E"]
        d = dev(c)
        rbf, cut = sentinel(E + 2, 64), sentinel(E + 2)
        shim.tn_edge_geom(E, d["e_vec"], nr, 64, T.WIDTH, T.RC, T.mu_of(nr), rbf, cut)
        sync()
        r = T.edge_geom_ref(c["e_vec"], nr)
        what = f"E={E} nr={nr}"
        check("edge_geom rbf", "edge_geom", rbf[:E], r["rbf"], what)  # columns past nr: scale 0, exactly 0
        check("edge_geom cut", "edge_geom", cut[:E], r["cut"], what)
        assert bool((rbf[E:] == SENT).all() and (cut[E:] == SENT).all()), f"rows past E written {what}"


# ------------------------------------------------------------------------------------------------ embedding
def embed_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    E = c["E"]
    cut = T.edge_geom_ref(c["e_vec"], 20)["cut"].x.float()
    return dict(U=T.rnd(g, T.N_ELEM, 64), V=T.rnd(g, T.N_ELEM, 64), P=T.rnd(g, E, 192), cut=cut, g=g)


@pytest.mark.parametrize("case", ["standard", "E_odd"])
def test_embed_agg_and_reverse(shim, case):
    c = std_graph(50) if case == "standard" else T.gen_graph(29, 51, E=259)
    n, E = c["n_own"], c["E"]
    assert case == "standard" or E % 8 != 0
    x = embed_inputs(c, 52)
    d = dev(c)
    U, V, P, cut = x["U"].cuda(), x["V"].cuda(), x["P"].cuda(), x["cut"].cuda()
    T0, nr0 = sentinel(n + 2, 10, 64), sentinel(n + 2, 64)
    shim.tn_embed_agg(n, d["row_ptr"], d["e_src"], d["type"], U, V, P, cut, d["e_vec"], T0, nr0)
    sync()
    gT0 = T.rnd(x["g"], n, 10, 64)  # with a component along the trace direction: the gvh formula must annihilate it
    gC0 = T.rnd(x["g"], E)
    r = T.embed_agg_ref(c, x["U"], x["V"], x["P"], x["cut"], gT0, gC0)
    check("embed_agg T0", "embed_agg", T0[:n], r["T0"], case)  # rows without edges: 0 exactly
    check("embed_agg nr0", "embed_agg", nr0[:n], r["nr0"], case)
    assert bool((T0[n:] == SENT).all() and (nr0[n:] == SENT).all()), f"rows past n_own written {case}"
    gP, gC, gvh = sentinel(E + 2, 192), gC0.cuda(), sentinel(E + 2, 3)
    shim.tn_embed_agg_bwd(E, d["e_src"], d["e_dst"], d["type"], U, V, P, cut, d["e_vec"], gT0.cuda(), gP, gC, gvh)
    sync()
    check("embed_agg_bwd gP", "embed_agg_bwd", gP[:E], r["gP"], case)
    check("embed_agg_bwd gC", "embed_agg_bwd", gC, r["gC"], case)
    check("embed_agg_bwd gvh", "embed_agg_bwd", gvh[:E], r["gvh"], case)
    assert bool((gP[E:] == SENT).all() and (gvh[E:] == SENT).all()), f"rows past E written {case}"


def test_edge_kernels_launch_nothing_at_zero(shim):
    """n_own = 0 and E = 0: nothing launched, nothing touched"""
    c = T.gen_graph(0, 5, n_halo=4)
    d = dev(c)
    z = torch.zeros(4, 192, device="cuda")
    bufs = [sentinel(4, 640) for _ in range(6)]
    cut, gC = sentinel(4), sentinel(4)
    shim.tn_edge_geom(0, d["e_vec"], 20, 64, T.WIDTH, T.RC, T.mu_of(20), bufs[0], cut)
    shim.tn_embed_agg(0, d["row_ptr"], d["e_src"], d["type"], z, z, z, z, z, bufs[1], bufs[2])
    shim.tn_embed_agg_bwd(0, d["e_src"], d["e_dst"], d["type"], z, z, z, z, z, z, bufs[3], gC, bufs[4])
    shim.tn_msg(0, d["row_ptr"], d["e_src"], z, z, z, bufs[5])
    shim.tn_msg_bwd(0, d["row_ptr"], d["e_src"], z, z, z, z, bufs[0], gC, bufs[1])
    F, vir = sentinel(4, 3), sentinel(9, dtype=torch.float64)
    shim.tn_edge_final(0, d["e_src"], d["e_dst"], d["e_vec"], d["gid"], 20, 64, T.WIDTH, T.RC, T.mu_of(20), z, z, z,
                       cut, F, vir, bufs[2])
    sync()
    for t in bufs + [cut, gC, F, vir]:
        assert bool((t == SENT).all()), "touched by an empty launch"


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("W", [64, 192])
def test_layernorm_and_reverse(shim, W):
    g = torch.Generator().manual_seed(60 + W)
    rows = 45  # % 8 != 0: the last block has warps without a row
    x = T.rnd(g, rows, W, s=2.0) + T.rnd(g, rows, 1)
    x[7] = 3.0 + 1e-4 * torch.randn(W, generator=g)  # nearly constant: the variance is below eps
    gamma, beta, gy = 1 + 0.3 * T.rnd(g, W), T.rnd(g, W, s=0.5), T.rnd(g, rows, W)
    y, st = sentinel(rows + 2, W), sentinel(rows + 2, 2)
    shim.tn_layernorm(rows, W, x.cuda(), gamma.cuda(), beta.cuda(), y, st)
    sync()
    r = T.layernorm_ref(x, gamma, beta, gy)
    check("layernorm y", "layernorm", y[:rows], r["y"], f"W={W}")
    check("layernorm stats", "layernorm", st[:rows], r["stats"], f"W={W}")
    assert bool((y[rows:] == SENT).all() and (st[rows:] == SENT).all())
    gx = sentinel(rows + 2, W)
    shim.tn_layernorm_bwd(rows, W, x.cuda(), st, gamma.cuda(), gy.cuda(), gx)
    sync()
    check("layernorm_bwd gx", "layernorm_bwd", gx[:rows], r["gx"], f"W={W}")
    assert bool((gx[rows:] == SENT).all())


# ------------------------------------------------------------------------------------------------ element-wise node ops
NODE_N = [1, 37, 300]  # 37 * 64 % 256 != 0: a partial last block


@pytest.mark.parametrize("n", NODE_N)
def test_scale_and_reverse(shim, n):
    g = torch.Generator().manual_seed(70 + n)
    X = T.gen_dec(g, n)
    Xh, q = sentinel(n + 1, 10, 64), sentinel(n + 1, 64)
    shim.tn_scale(n, X.cuda(), Xh, q)
    sync()
    r = T.node_ref("scale", n, [X])
    check("scale Xh", "node", Xh[:n], r["Xh"], f"n={n}")
    check("scale q", "node", q[:n], r["q"], f"n={n}")
    assert bool((Xh[n:] == SENT).all() and (q[n:] == SENT).all())
    gXh = T.rnd(g, n, 10, 64)
    gb = torch.cat([gXh, torch.full((1, 10, 64), SENT)]).cuda()
    shim.tn_scale_bwd(n, X.cuda(), q, gb)
    sync()
    check_adj("scale_bwd gX", "node_bwd", gb[:n], T.node_ref("scale", n, [X], gXh)["gX"], n, f"n={n}")
    assert bool((gb[n:] == SENT).all())


@pytest.mark.parametrize("so3", [0, 1], ids=["O3", "SO3"])
@pytest.mark.parametrize("n", NODE_N)
def test_prod_and_reverse(shim, n, so3):
    g = torch.Generator().manual_seed(80 + n + so3)
    m, Y = T.gen_dec(g, n), T.gen_dec(g, n)
    Pn = sentinel(n + 1, 10, 64)
    shim.tn_prod(n, m.cuda(), Y.cuda(), so3, Pn)
    sync()
    check("prod Pn", "node", Pn[:n], T.node_ref("prod", n, [m, Y], so3=so3)["Pn"], f"n={n} so3={so3}")
    assert bool((Pn[n:] == SENT).all())
    gPn = T.rnd(g, n, 10, 64)
    gm, gY = sentinel(n + 1, 10, 64), sentinel(n + 1, 10, 64)
    shim.tn_prod_bwd(n, m.cuda(), Y.cuda(), so3, gPn.cuda(), gm, gY)
    sync()
    r = T.node_ref("prod", n, [m, Y], gPn, so3=so3)
    check_adj("prod_bwd gmsg", "node_bwd", gm[:n], r["gmsg"], n, f"n={n} so3={so3}")
    check_adj("prod_bwd gY", "node_bwd", gY[:n], r["gY"], n, f"n={n} so3={so3}")
    assert bool((gm[n:] == SENT).all() and (gY[n:] == SENT).all())


@pytest.mark.parametrize("n", NODE_N)
def test_update_and_reverse(shim, n):
    g = torch.Generator().manual_seed(90 + n)
    Xh, dX = T.gen_dec(g, n), T.gen_dec(g, n)
    Xn = sentinel(n + 1, 10, 64)
    shim.tn_update(n, Xh.cuda(), dX.cuda(), Xn)
    sync()
    check("update Xn", "node", Xn[:n], T.node_ref("update", n, [Xh, dX])["Xn"], f"n={n}")
    gXn = T.rnd(g, n, 10, 64)
    gdX = sentinel(n + 1, 10, 64)
    shim.tn_update_bwd(n, dX.cuda(), gXn.cuda(), gdX)
    sync()
    check_adj("update_bwd gdX", "node_bwd", gdX[:n], T.node_ref("update", n, [Xh, dX], gXn)["gdX"], n, f"n={n}")
    assert bool((Xn[n:] == SENT).all() and (gdX[n:] == SENT).all())


@pytest.mark.parametrize("n", NODE_N)
def test_invariants_and_reverse(shim, n):
    g = torch.Generator().manual_seed(100 + n)
    X = T.gen_dec(g, n)
    inv = sentinel(n + 1, 3, 64)
    shim.tn_invariants(n, X.cuda(), inv)
    sync()
    check("invariants inv", "node", inv[:n], T.node_ref("invariants", n, [X])["inv"], f"n={n}")
    ginv = T.rnd(g, n, 3, 64)
    gX = sentinel(n + 1, 10, 64)
    shim.tn_invariants_bwd(n, X.cuda(), ginv.cuda(), gX)
    sync()
    check_adj("invariants_bwd gX", "node_bwd", gX[:n], T.node_ref("invariants", n, [X], ginv)["gX"], n, f"n={n}")
    assert bool((inv[n:] == SENT).all() and (gX[n:] == SENT).all())


@pytest.mark.parametrize("n", NODE_N)
def test_embed_out_and_reverse(shim, n):
    g = torch.Generator().manual_seed(110 + n)
    T0m, s2p = T.gen_dec(g, n), T.rnd(g, n, 192, s=2.0)
    X0 = sentinel(n + 1, 10, 64)
    shim.tn_embed_out(n, T0m.cuda(), s2p.cuda(), X0)
    sync()
    check("embed_out X0", "node", X0[:n], T.node_ref("embed_out", n, [T0m, s2p])["X0"], f"n={n}")
    gX0 = T.rnd(g, n, 10, 64)
    gT0m, gs2p = sentinel(n + 1, 10, 64), sentinel(n + 1, 192)
    shim.tn_embed_out_bwd(n, T0m.cuda(), s2p.cuda(), gX0.cuda(), gT0m, gs2p)
    sync()
    r = T.node_ref("embed_out", n, [T0m, s2p], gX0)
    check_adj("embed_out_bwd gT0m", "node_bwd", gT0m[:n], r["gT0m"], n, f"n={n}")
    check("embed_out_bwd gs2p", "node_bwd", gs2p[:n], r["gs2p"], f"n={n}")
    assert bool((X0[n:] == SENT).all() and (gT0m[n:] == SENT).all() and (gs2p[n:] == SENT).all())


@pytest.mark.parametrize("n", NODE_N)
def test_norm_bwd_add(shim, n):
    g = torch.Generator().manual_seed(120 + n)
    T0, gnr0 = T.gen_dec(g, n), T.rnd(g, n, 64)
    p0 = torch.cat([T.gen_dec(g, n), torch.full((1, 10, 64), SENT)])
    gT0 = p0.cuda()
    shim.tn_norm_bwd_add(n, T0.cuda(), gnr0.cuda(), gT0)
    sync()
    r = T.node_ref("norm", n, [T0], gnr0)["gT0"]
    pre = T.mproj(KU.Mag(T.d64(p0[:n])), n)
    check_adj("norm_bwd_add gT0", "node_bwd", gT0[:n], KU.Mag(pre.x + r.x, pre.s + r.s), n, f"n={n}")
    same("norm_bwd_add rows past n", gT0[n:], p0[n:])


# ------------------------------------------------------------------------------------------------ message
@pytest.mark.parametrize("case", ["standard", "E_odd"])
def test_msg_and_reverse(shim, case):
    c = std_graph(130) if case == "standard" else T.gen_graph(29, 131, E=259)
    n, nl, E = c["n_own"], c["n_loc"], c["E"]
    g = torch.Generator().manual_seed(132)
    f3p = T.rnd(g, E, 192, s=2.0)
    cut = T.edge_geom_ref(c["e_vec"], 20)["cut"].x.float()
    Y = T.gen_dec(g, nl)
    d = dev(c)
    out = sentinel(n + 1, 10, 64)
    shim.tn_msg(n, d["row_ptr"], d["e_src"], f3p.cuda(), cut.cuda(), Y.cuda(), out)
    sync()
    check("msg msg", "msg", out[:n], T.msg_ref(c, f3p, cut, Y)["msg"], case)  # rows without edges: 0 exactly
    assert bool((out[n:] == SENT).all())
    # reverse: gY owned rows prefilled (as prod_bwd leaves them), halo rows too; red.add into source rows only
    gmsg, gC0, gY0 = T.rnd(g, n, 10, 64), T.rnd(g, E), T.rnd(g, nl, 10, 64)
    g3, gC, gY = sentinel(E + 1, 192), gC0.cuda(), gY0.cuda()
    shim.tn_msg_bwd(n, d["row_ptr"], d["e_src"], f3p.cuda(), cut.cuda(), Y.cuda(), gmsg.cuda(), g3, gC, gY)
    sync()
    r = T.msg_ref(c, f3p, cut, Y, gmsg, gC0, gY0)
    check("msg_bwd g3", "msg_bwd", g3[:E], r["g3"], case)
    check("msg_bwd gC", "msg_bwd", gC, r["gC"], case)
    hit = torch.zeros(nl, dtype=torch.bool)
    hit[c["e_src"].long()] = True
    assert bool(hit[c["n_own"]:].any()), "no halo source"
    check_adj("msg_bwd gY", "msg_bwd", gY[hit.cuda()], KU.Mag(r["gY"].x[hit], r["gY"].s[hit]), int(hit.sum()), case)
    same("gY rows that are no source", gY[(~hit).cuda()], gY0[~hit], case)
    assert bool((g3[E:] == SENT).all())


# ------------------------------------------------------------------------------------------------ readout
@pytest.mark.parametrize("wgt", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("atomic", [False, True], ids=["noatom", "atom_e"])
@pytest.mark.parametrize("eref", [False, True], ids=["noeref", "eref"])
@pytest.mark.parametrize("W", [64, 128])
def test_readout_final(shim, W, eref, atomic, wgt):
    c = T.gen_graph(37, 140 + W + 2 * eref + 4 * atomic + 8 * wgt)
    g, n, N = c["g"], c["n_own"], c["N"]
    hL, hG = T.rnd(g, n, W), T.rnd(g, n, W)
    wL, wG = T.rnd(g, W, s=W ** -0.5), T.rnd(g, W, s=W ** -0.5)
    er = torch.linspace(-3.0, -1.0, T.N_ELEM, dtype=torch.float64) if eref else None
    wv = (0.5 + torch.rand(N, generator=g)) if wgt else None
    lout, gout, ea = sentinel(n + 1), sentinel(n + 1), sentinel(n + 1)
    energy = torch.full((1,), 0.25, dtype=torch.float64, device="cuda")
    ae = sentinel(N, dtype=torch.float64) if atomic else None
    shim.tn_readout_final(n, W, hL.cuda(), wL.cuda(), 0.3, hG.cuda(), wG.cuda(), -0.2, c["type"].cuda(),
                          None if er is None else er.cuda(), 1.3, lout, gout, ea, energy, c["gid"].cuda(), ae, 0.07,
                          None if wv is None else wv.cuda())
    sync()
    r = T.readout_final_ref(c, n, W, hL, wL, 0.3, hG, wG, -0.2, er, 1.3, 0.07 if atomic else 0.0, wv,
                            torch.tensor([0.25], dtype=torch.float64))
    what = f"W={W} eref={eref} atomic={atomic} wgt={wgt}"
    for k, o in (("lout", lout), ("gout", gout), ("e_atom", ea)):
        check(f"readout_final {k}", "readout", o[:n], r[k], what)
        assert bool((o[n:] == SENT).all())
    check("readout_final energy", "readout", energy, r["energy"], what)
    if atomic:
        gid = c["gid"][:n].long()
        check("readout_final atom_e", "readout", ae[gid.cuda()], r["atom_e"], what)
        free = torch.ones(N, dtype=torch.bool)
        free[gid] = False
        assert bool((ae.cpu()[free] == SENT).all()), f"atom_e of other atoms written {what}"


@pytest.mark.parametrize("wgt", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("W", [64, 128])
def test_readout_seed(shim, W, wgt):
    c = T.gen_graph(37, 150 + W + wgt)
    g, n, N = c["g"], c["n_own"], c["N"]
    lout, gout = T.rnd(g, n), 0.02 + 0.96 * torch.rand(n, generator=g)
    wL, wG = T.rnd(g, W, s=W ** -0.5), T.rnd(g, W, s=W ** -0.5)
    preL, preG = T.rnd(g, n, W, s=2.0), T.rnd(g, n, W, s=2.0)
    wv = (0.5 + torch.rand(N, generator=g)) if wgt else None
    gL, gG = sentinel(n + 1, W), sentinel(n + 1, W)
    shim.tn_readout_seed(n, W, lout.cuda(), gout.cuda(), 1.3, wL.cuda(), wG.cuda(), preL.cuda(), preG.cuda(), gL, gG,
                         c["gid"].cuda(), None if wv is None else wv.cuda())
    sync()
    r = T.readout_seed_ref(c, n, lout, gout, 1.3, wL, wG, preL, preG, wv)
    check("readout_seed gL", "readout", gL[:n], r["gL"], f"W={W} wgt={wgt}")
    check("readout_seed gG", "readout", gG[:n], r["gG"], f"W={W} wgt={wgt}")
    assert bool((gL[n:] == SENT).all() and (gG[n:] == SENT).all())


# ------------------------------------------------------------------------------------------------ edge final
def run_graph(seed):
    """runs of equal destinations of length 1, across lane 32 (edges 20..39), longer than 64 (edges 70..159) and across
    the 256-thread boundary (edges 220..269); E = 306, not a multiple of 32"""
    counts = [1, 1, 1, 17, 20, 25, 5, 90] + [1] * 10 + [50, 50, 30, 1, 2, 3]
    return T.gen_graph(len(counts), seed, counts=counts)


@pytest.mark.parametrize("atomic", [False, True], ids=["noatom", "atom_vir"])
@pytest.mark.parametrize("nr", [1, 32, 64])
def test_edge_final(shim, nr, atomic):
    for c in (std_graph(160 + nr), run_graph(161 + nr)):
        g, E, N = c["g"], c["E"], c["N"]
        assert E % 32 != 0
        d = dev(c)
        g_rbf = T.rnd(g, E, 64, s=0.5)
        g_rbf[:, nr:] = float("nan")  # padding columns are never read
        gC, gvh = T.rnd(g, E), T.rnd(g, E, 3)
        F0, v0, av0 = T.rnd(g, N, 3), T.rnd(g, 9).double(), T.rnd(g, N, 12)
        F, vir = F0.cuda(), v0.cuda()
        av = av0.cuda() if atomic else None
        gd = sentinel(E + 1)
        shim.tn_edge_final(E, d["e_src"], d["e_dst"], d["e_vec"], d["gid"], nr, 64, T.WIDTH, T.RC, T.mu_of(nr),
                           g_rbf.cuda(), gC.cuda(), gvh.cuda(), gd, F, vir, av)
        sync()
        r = T.edge_final_ref(c, nr, g_rbf, gC, gvh, F0, v0, av0 if atomic else None)
        what = f"E={E} nr={nr}"
        check("edge_final gd", "edge_final", gd[:E], r["gd"], what)
        assert bool((gd[E:] == SENT).all())
        check("edge_final forces", "edge_final", F, r["forces"], what)
        check("edge_final virial", "edge_final", vir, r["virial"], what)
        if atomic:
            ref = KU.Mag(r["atom_vir"].x[:, :9], r["atom_vir"].s[:, :9])
            check("edge_final atom_vir", "edge_final", av[:, :9], ref, what)
            same("atom_vir pitch columns 9..11", av[:, 9:], av0[:, 9:], what)
        hit = torch.zeros(N, dtype=torch.bool)
        hit[c["gid"].long()[c["e_src"].long()]] = True
        hit[c["gid"].long()[c["e_dst"].long()]] = True
        same("forces of atoms without edges", F[(~hit).cuda()], F0[~hit], what)
