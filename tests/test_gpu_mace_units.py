"""Each MACE launcher of kernels_mace.cu on its own, called through tests/kernel_shim.cu on synthetic inputs that meet
the engine's contract (tests/mace_units_ref.py), against a float64 restatement built from the project's MACE oracles.

Every element must satisfy |out - ref| <= tol * scale (the first-order rounding bound of mace_units_ref.py); columns a
kernel zero-fills have scale 0 and so must be exactly 0 (Y for k >= nsh, eb for n >= nb); rows, planes and columns a
launch must not write keep their sentinels or prefills bit for bit.  The cases aim at partial last blocks, E = 1 and
E = 257 for the per-edge kernels, n_own = 0 and E = 0 (nothing launched, nothing touched), atoms without edges, a row
of 300 edges, halo sources (the reverse's atomics landing in halo rows), a self-image edge, a channel pitch wider than
the model's channels (padding that must stay zero), every model shape the engine accepts and every option
(Agnesi / ZBL, atom_e, atom_vir, heat-flux weights).

B2M_MACE_UNITS_REPORT=<path> writes the largest normalised error of every launcher output to <path> (JSON).
"""
import json
import os

import pytest
import torch

from tests import kernel_units_ref as KU
from tests import mace_units_ref as M
from tests.mace_units_ref import ST, call

pytestmark = pytest.mark.gpu
ERRS = {}
CH = [(32, 64), (96, 128)]  # (model channels, row pitch)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = KU.Shim(KU.build_shim(tmp_path_factory.mktemp("kernel_shim")))
    yield s
    path = os.environ.get("B2M_MACE_UNITS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({k: ERRS[k] for k in sorted(ERRS)}, f, indent=1)
    for k in sorted(ERRS):
        print(f"mace-units max |out - ref| / scale  {k:<26s} {ERRS[k]:.3e}")


def check(key, tol, out, ref, what=""):
    KU.check(ERRS, key, M.TOL[tol], out, ref, what)


def same(name, out, before, what=""):
    """out equals before bit for bit"""
    o, b = out.detach().cpu().contiguous(), before.detach().cpu().contiguous()
    assert torch.equal(o.view(-1).view(torch.int32 if o.dtype == torch.float32 else torch.int64),
                       b.view(-1).view(torch.int32 if b.dtype == torch.float32 else torch.int64)), f"{name} {what} changed"


def dev(c):
    return {k: v.cuda() for k, v in c.items() if isinstance(v, torch.Tensor)}


def sync():
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ edge geometry
def graph_cases(seed):
    """the standard graph (atoms without edges, a 300-edge row, halo sources), E = 1 and E = 257"""
    return [M.gen_graph(37, seed, empty=3, heavy=300), M.gen_graph(5, seed + 1, E=1), M.gen_graph(29, seed + 2, E=257)]


def radial_args(nb):
    w, pref = M.radial_params(nb)
    return [nb, M.P_CUT, float(M.R_MAX), pref, w]


def core_args(core):
    return [core["elem"].cuda(), core["zbl"], core["agnesi"], core["zp"], core["cf"]]


@pytest.mark.parametrize("agnesi", [False, True], ids=["plain", "agnesi"])
@pytest.mark.parametrize("nb", [1, 8, 64])
def test_edge_geom(shim, nb, agnesi):
    core = M.core_params(False, agnesi)
    for c in graph_cases(nb + 3 * agnesi):
        d = dev(c)
        for nsh in (1, 4, 9, 16):
            E = c["E"]
            Y, eb = M.sentinel(E + 3, 16), M.sentinel(E + 3, 64)
            call(shim, "edge_geom", ST, M.ctypes.c_int64(E), d["e_vec"], *radial_args(nb), nsh, Y, eb, d["e_src"],
                 d["e_dst"], d["type"], *core_args(core))
            sync()
            ref = M.edge_geom_ref(c, nb, nsh, core)
            what = f"E={E} nsh={nsh}"
            check("edge_geom Y", "edge_geom", Y[:E], ref["Y"], what)
            check("edge_geom eb", "edge_geom", eb[:E], ref["eb"], what)
            assert bool((Y[E:] == M.SENTINEL).all() and (eb[E:] == M.SENTINEL).all()), f"rows past E written {what}"


def test_edge_kernels_launch_nothing_at_zero(shim):
    """E = 0 and n_own = 0: nothing launched, nothing touched"""
    c = M.gen_graph(0, 5, n_halo=4)
    d = dev(c)
    core = M.core_params(True, True)
    Y, eb, el = M.sentinel(4, 16), M.sentinel(4, 64), M.sentinel(4)
    call(shim, "edge_geom", ST, M.ctypes.c_int64(0), d["e_vec"], *radial_args(8), 16, Y, eb, d["e_src"], d["e_dst"],
         d["type"], *core_args(core))
    call(shim, "zbl", ST, 0, d["row_ptr"], d["e_src"], d["e_vec"], d["type"], *core_args(core), el)
    F, vir, av = M.sentinel(4, 3), M.sentinel(9, dtype=torch.float64), M.sentinel(4, 12)
    call(shim, "edge_final", ST, M.ctypes.c_int64(0), 16, d["e_src"], d["e_dst"], d["e_vec"], d["gid"], d["type"],
         *radial_args(8), *core_args(core), Y, Y, F, vir, av, None)
    h, A = M.sentinel(4, 64), M.sentinel(16, 4, 64)
    call(shim, "embed", ST, 0, 64, d["type"], h, h)
    call(shim, "msg", 0, ST, 0, 64, 4, d["row_ptr"], d["e_src"], A, A, A, A, None, None, None, None)
    call(shim, "readout_seed", ST, 0, 64, 16, h, h, h, 1.0, A, d["gid"], None)
    sync()
    for name, t in (("Y", Y), ("eb", eb), ("e_lin", el), ("forces", F), ("virial", vir), ("atom_vir", av), ("h", h),
                    ("A", A)):
        assert bool((t == M.SENTINEL).all()), f"{name} touched by an empty launch"


@pytest.mark.parametrize("zbl_case", ["standard", "E257"])
def test_zbl(shim, zbl_case):
    c = M.gen_graph(37, 11, empty=3, heavy=300) if zbl_case == "standard" else M.gen_graph(29, 12, E=257)
    core = M.core_params(True, False)
    d = dev(c)
    n = c["n_own"]
    el0 = M.rnd(c["g"], n + 3)
    el0[n:] = M.SENTINEL
    el = el0.cuda()
    call(shim, "zbl", ST, n, d["row_ptr"], d["e_src"], d["e_vec"], d["type"], *core_args(core), el)
    sync()
    check("zbl e_lin", "zbl", el[:n], M.zbl_ref(c, core, el0[:n]), zbl_case)
    same("e_lin rows past n_own", el[n:], el0[n:])


def test_embed(shim):
    c = M.gen_graph(37, 13)
    for Cr, C in CH:
        W = M.rnd(c["g"], len(M.ELEMS), C, Cr=Cr)
        n = c["n_loc"]
        h = M.sentinel(n * C + 64)
        call(shim, "embed", ST, n, C, c["type"].cuda(), W.cuda(), h)
        sync()
        same("embed", h[: n * C], W[c["type"].long()].reshape(-1))
        assert bool((h[n * C:] == M.SENTINEL).all())


# ------------------------------------------------------------------------------------------------ messages
def msg_inputs(c, C, Cr, RW, seed):
    g = torch.Generator().manual_seed(seed)
    E, n = c["E"], c["n_own"]
    nsh = 16
    v = M.d64(c["e_vec"][:, :3])
    Y = M.sh(v, nsh).float() if E else torch.zeros(0, 16)
    return dict(R=M.rnd(g, E, RW // C, C, Cr=Cr).reshape(E, RW), Y=Y, g=g)


@pytest.mark.parametrize("Cr,C", CH)
@pytest.mark.parametrize("L1", [1, 2, 3, 4])
def test_msg_and_reverse(shim, L1, Cr, C):
    c = M.gen_graph(37, 20 + L1, empty=3, heavy=300)
    nsh, n, nl, E = L1 * L1, c["n_own"], c["n_loc"], c["E"]
    x = msg_inputs(c, C, Cr, L1 * C, 100 + L1)
    g = x["g"]
    Y = x["Y"].clone()
    Y[:, nsh:] = torch.randn(E, 16 - nsh, generator=g)  # columns past nsh are never read
    u = M.rnd(g, nl, C, Cr=Cr)
    d = dev(c)
    A = M.sentinel(16, n, C)
    call(shim, "msg", 0, ST, n, C, L1, d["row_ptr"], d["e_src"], x["R"].cuda(), Y.cuda(), u.cuda(), A, None, None, None,
         None)
    sync()
    f = M.msg_fn(c, C, L1)
    ref = M.multilinear(f, dict(R=x["R"], Y=Y, u=u))
    what = f"L1={L1} C={Cr}/{C}"
    check("msg A", "msg", A[:nsh], M.KU_mag(ref, (nsh, n, C)), what)
    assert bool((A[nsh:] == M.SENTINEL).all()), f"planes k >= nsh of A written {what}"
    # reverse on the first n - 4 rows: gR = for their edges only; gY += (column 0 included); gu += (halo rows too)
    nb_ = n - 4
    cb = M.restrict(c, nb_)
    Eb = cb["E"]
    gA = M.rnd(g, nsh, nb_, C, Cr=Cr)
    gR = M.sentinel(E, L1 * C)
    gY0, gu0 = M.rnd(g, E, 16), M.rnd(g, nl, C)
    gY, gu = gY0.cuda(), gu0.cuda()
    call(shim, "msg", 1, ST, nb_, C, L1, d["row_ptr"], d["e_src"], x["R"].cuda(), Y.cuda(), u.cuda(), None, gA.cuda(),
         gR, gY, gu)
    sync()
    fb = M.msg_fn(cb, C, L1)
    r = M.multilinear(fb, dict(R=x["R"][:Eb], Y=Y[:Eb], u=u), g=gA, wrt=("R", "Y", "u"))
    check("msg_bwd gR", "msg_bwd", gR[:Eb], r["R"], what)
    assert bool((gR[Eb:] == M.SENTINEL).all()), f"gR of edges outside the launch written {what}"
    check("msg_bwd gY", "msg_bwd", gY[:Eb, :nsh], M.plus(gY0[:Eb, :nsh], r["Y"][:, :nsh]), what)
    same("gY columns past nsh", gY[:, nsh:], gY0[:, nsh:], what)
    same("gY of edges outside the launch", gY[Eb:], gY0[Eb:], what)
    check("msg_bwd gu", "msg_bwd", gu, M.plus(gu0, r["u"]), what)


@pytest.mark.parametrize("Cr,C", CH)
@pytest.mark.parametrize("max_ell", [1, 2, 3])
def test_msg_eq_and_reverse(shim, max_ell, Cr, C):
    c = M.gen_graph(37, 40 + max_ell, empty=3, heavy=300)
    paths, per, base, nslots = M.eq_layout(max_ell)
    NP, nsh, n, nl, E = len(paths), (max_ell + 1) ** 2, c["n_own"], c["n_loc"], c["E"]
    x = msg_inputs(c, C, Cr, NP * C, 200 + max_ell)
    g = x["g"]
    Y = x["Y"].clone()
    Y[:, nsh:] = torch.randn(E, 16 - nsh, generator=g)
    u = M.rnd(g, nl, 4, C, Cr=Cr).reshape(nl, 4 * C)
    d = dev(c)
    Am = M.sentinel(nslots * n * C + 64)
    call(shim, "msg_eq", 0, ST, max_ell, n, C, d["row_ptr"], d["e_src"], x["R"].cuda(), Y.cuda(), u.cuda(), Am, None,
         None, None)
    sync()
    ref = M.multilinear(M.msg_eq_fn(c, C, max_ell), dict(R=x["R"], Y=Y, u=u))
    what = f"max_ell={max_ell} C={Cr}/{C}"
    check("msg_eq Am", "msg_eq", Am[: nslots * n * C], ref, what)
    assert bool((Am[nslots * n * C:] == M.SENTINEL).all()), f"Am written past its slots {what}"
    nb_ = n - 4
    cb = M.restrict(c, nb_)
    Eb = cb["E"]
    gAm = M.rnd(g, nslots, nb_, C)
    gAm.view(-1, C)[:, Cr:] = 0.0
    Rb = x["R"].clone().cuda()
    gY0, gu0 = M.rnd(g, E, 16), M.rnd(g, nl, 4 * C)
    gY, gu = gY0.cuda(), gu0.cuda()
    call(shim, "msg_eq", 1, ST, max_ell, nb_, C, d["row_ptr"], d["e_src"], Rb, Y.cuda(), u.cuda(), None, gAm.cuda(), gY,
         gu)
    sync()
    r = M.multilinear(M.msg_eq_fn(cb, C, max_ell), dict(R=x["R"][:Eb], Y=Y[:Eb], u=u), g=gAm.reshape(-1),
                      wrt=("R", "Y", "u"))
    check("msg_eq_bwd gR (over R)", "msg_eq_bwd", Rb[:Eb], r["R"], what)
    same("R of edges outside the launch", Rb[Eb:], x["R"][Eb:], what)
    check("msg_eq_bwd gY", "msg_eq_bwd", gY[:Eb, 1:nsh], M.plus(gY0[:Eb, 1:nsh], r["Y"][:, 1:nsh]), what)
    same("gY column 0 (Y[0] = 1 carries no gradient)", gY[:, 0], gY0[:, 0], what)
    same("gY columns past nsh", gY[:, nsh:], gY0[:, nsh:], what)
    same("gY of edges outside the launch", gY[Eb:], gY0[Eb:], what)
    check("msg_eq_bwd gu", "msg_eq_bwd", gu, M.plus(gu0, r["u"]), what)


# ------------------------------------------------------------------------------------------------ element mixes
@pytest.mark.parametrize("accum", [False, True], ids=["set", "accum"])
@pytest.mark.parametrize("nsh", [1, 16])
@pytest.mark.parametrize("Cr,C", CH)
def test_elem_mix(shim, nsh, accum, Cr, C):
    c = M.gen_graph(37, 60 + nsh)
    g, n, L1 = c["g"], c["n_own"], 4
    Lw = 1 if nsh == 1 else L1
    W = M.rnd(g, len(M.ELEMS), Lw, C, C, s=C ** -0.5, Cr=Cr)
    W[..., Cr:, :] = 0.0
    x = M.rnd(g, nsh, n, C, Cr=Cr)
    out0 = M.rnd(g, nsh * n * C + 64)
    out0[nsh * n * C:] = M.SENTINEL
    out = out0.cuda()
    call(shim, "elem_mix", ST, n, C, L1, nsh, c["type"].cuda(), W.cuda(), x.cuda(), out, int(accum))
    sync()
    r = M.multilinear(M.elem_mix_fn(c, n, C, L1, nsh), dict(W=W, x=x))
    if accum:
        r = M.plus(out0[: nsh * n * C], r.x.reshape(-1), r.s.reshape(-1))
    check("elem_mix out", "elem_mix", out[: nsh * n * C], M.flat(r), f"nsh={nsh} accum={accum} C={Cr}/{C}")
    same("elem_mix tail", out[nsh * n * C:], out0[nsh * n * C:])


@pytest.mark.parametrize("accum", [False, True], ids=["set", "accum"])
@pytest.mark.parametrize("ncomp", [1, 4])
@pytest.mark.parametrize("Cr,C", CH)
def test_elem_mix_rows(shim, ncomp, accum, Cr, C):
    c = M.gen_graph(37, 70 + ncomp)
    g, n = c["g"], c["n_own"]
    Lw = 2 if ncomp == 4 else 1
    ldi, ldo = 4 * C + 64, 4 * C
    W = M.rnd(g, len(M.ELEMS), Lw, C, C, s=C ** -0.5, Cr=Cr)
    W[..., Cr:, :] = 0.0
    x = M.rnd(g, n, ldi)
    x[:, : 4 * C].unflatten(1, (4, C))[..., Cr:] = 0.0
    out0 = M.rnd(g, n + 2, ldo)
    out = out0.cuda()
    call(shim, "elem_mix_rows", ST, n, C, ncomp, ldi, ldo, c["type"].cuda(), W.cuda(), x.cuda(), out, int(accum))
    sync()
    r = M.multilinear(M.elem_mix_rows_fn(c, n, C, ncomp, ldi), dict(W=W, x=x))
    if accum:
        r = M.plus(out0[:n, : ncomp * C], r.x, r.s)
    check("elem_mix_rows out", "elem_mix", out[:n, : ncomp * C], r, f"ncomp={ncomp} accum={accum} C={Cr}/{C}")
    same("elem_mix_rows other columns", out[:n, ncomp * C:], out0[:n, ncomp * C:])
    same("elem_mix_rows rows past n", out[n:], out0[n:])


# ------------------------------------------------------------------------------------------------ symmetric contraction
def run_symc(shim, max_ell, corr, eq, Cr, C, seed):
    c = M.gen_graph(37, seed)
    g, n, nsh = c["g"], c["n_own"], (max_ell + 1) ** 2
    mods = M.make_contraction(max_ell, corr, Cr, eq, seed)
    terms = M.build_terms(shim, mods, nsh)
    w, _ = M.stack_weights(mods, C)
    Ktot = w.shape[1]
    A = M.rnd(g, nsh, n, C, s=0.7, Cr=Cr)
    nB = 4 if eq else 1
    B = M.sentinel(nB * n * C + 64)
    t = c["type"].cuda()
    call(shim, "symc", int(eq), 0, ST, n, C, nsh, Ktot, t, A.cuda(), terms.cuda(), len(terms), w.cuda(), None, B)
    sync()
    f = M.symc_fn(mods, c, n, C, nsh, eq)
    what = f"max_ell={max_ell} corr={corr} C={Cr}/{C}"
    key = "symc_eq" if eq else "symc"
    check(f"{key} B", "symc", B[: nB * n * C], M.multilinear(f, dict(A=A)), what)
    assert bool((B[nB * n * C:] == M.SENTINEL).all()), f"B written past its planes {what}"
    gB = M.rnd(g, nB, n, C, Cr=Cr)
    gA = M.sentinel(16, n, C)
    call(shim, "symc", int(eq), 1, ST, n, C, nsh, Ktot, t, A.cuda(), terms.cuda(), len(terms), w.cuda(), gB.cuda(), gA)
    sync()
    r = M.multilinear(f, dict(A=A), g=gB.reshape(-1), wrt=("A",))
    check(f"{key}_bwd gA", "symc_bwd", gA[:nsh], M.KU_mag(r["A"], (nsh, n, C)), what)
    assert bool((gA[nsh:] == M.SENTINEL).all()), f"planes k >= nsh of gA written {what}"


@pytest.mark.parametrize("corr", [1, 2, 3])
@pytest.mark.parametrize("max_ell", [0, 1, 2, 3])
def test_symc(shim, max_ell, corr):
    Cr, C = CH[(max_ell + corr) % 2]
    run_symc(shim, max_ell, corr, False, Cr, C, 300 + 10 * max_ell + corr)


@pytest.mark.parametrize("max_ell,corr", [(1, 1), (1, 3), (2, 2), (3, 3)])
def test_symc_eq(shim, max_ell, corr):
    Cr, C = CH[max_ell % 2]
    run_symc(shim, max_ell, corr, True, Cr, C, 400 + 10 * max_ell + corr)


# ------------------------------------------------------------------------------------------------ readouts
def test_readout_lin(shim):
    for Cr, C in CH:
        c = M.gen_graph(37, 80 + C)
        g, n = c["g"], c["n_own"]
        ld = 4 * C
        h = M.rnd(g, n, ld)
        w = M.rnd(g, C, s=C ** -0.5, Cr=Cr)
        el0 = M.rnd(g, n + 3)
        el = el0.cuda()
        call(shim, "readout_lin", ST, n, C, ld, h.cuda(), w.cuda(), el)
        sync()
        r = M.multilinear(lambda a, h, w: h[:, :C] @ w, dict(h=h, w=w))
        check("readout_lin e_lin", "readout", el[:n], M.plus(el0[:n], r.x, r.s), f"C={C}")
        same("e_lin rows past n_own", el[n:], el0[n:])


@pytest.mark.parametrize("wgt", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("atomic", [False, True], ids=["noatom", "atom_e"])
@pytest.mark.parametrize("H", [1, 16, 256])
def test_readout_final(shim, H, atomic, wgt):
    Cr, C = CH[H % 2]
    c = M.gen_graph(37, 90 + H)
    g, n, N = c["g"], c["n_own"], c["N"]
    h = M.rnd(g, n, C, Cr=Cr)
    W1 = M.rnd(g, C, H, s=C ** -0.5)
    W1[Cr:] = 0.0
    w2 = M.rnd(g, H, s=1.6 * H ** -0.5)
    el = M.rnd(g, n)
    E0 = torch.linspace(-3.0, -1.0, len(M.ELEMS), dtype=torch.float64)
    wv = (0.5 + torch.rand(N, generator=g)) if wgt else None
    pre = M.sentinel(n + 2, H)
    energy = torch.full((1,), 0.25, dtype=torch.float64, device="cuda")
    ae = M.sentinel(N, dtype=torch.float64) if atomic else None
    call(shim, "readout_final", ST, n, C, H, h.cuda(), W1.cuda(), w2.cuda(), el.cuda(), c["type"].cuda(), E0.cuda(),
         M.ctypes.c_double(1.3), M.ctypes.c_double(-0.2), pre, energy, c["gid"].cuda(), ae,
         None if wv is None else wv.cuda())
    sync()
    r = M.readout_final_ref(c, h, W1, w2, el, E0, 1.3, -0.2, wv)
    what = f"H={H} atomic={atomic} wgt={wgt}"
    check("readout_final pre", "readout", pre[:n], r["pre"], what)
    assert bool((pre[n:] == M.SENTINEL).all())
    check("readout_final energy", "readout", energy, M.plus(torch.tensor([0.25]), r["energy"].x, r["energy"].s), what)
    if atomic:
        gid = c["gid"][:n].long()
        check("readout_final atom_e", "readout", ae[gid.cuda()], r["eps"], what)
        free = torch.ones(N, dtype=torch.bool)
        free[gid] = False
        assert bool((ae.cpu()[free] == M.SENTINEL).all()), f"atom_e of other atoms written {what}"


@pytest.mark.parametrize("wgt", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("H", [1, 16, 256])
def test_readout_seed_and_add_row(shim, H, wgt):
    Cr, C = CH[H % 2]
    c = M.gen_graph(37, 110 + H)
    g, n, nl, N = c["g"], c["n_own"], c["n_loc"], c["N"]
    pre = M.rnd(g, n, H, s=2.0)
    W1 = M.rnd(g, C, H, s=C ** -0.5)
    W1[Cr:] = 0.0
    w2 = M.rnd(g, H, s=1.6 * H ** -0.5)
    wv = (0.5 + torch.rand(N, generator=g)) if wgt else None
    wd = None if wv is None else wv.cuda()
    gh = M.sentinel(nl, C)
    call(shim, "readout_seed", ST, n, C, H, pre.cuda(), W1.cuda(), w2.cuda(), 1.3, gh, c["gid"].cuda(), wd)
    sync()
    what = f"H={H} wgt={wgt}"
    check("readout_seed gh", "readout", gh[:n], M.readout_seed_ref(c, pre, W1, w2, 1.3, wv), what)
    assert bool((gh[n:] == M.SENTINEL).all()), f"halo rows of gh written {what}"
    # add_row: gh[i][c] += scale wgt w[c] on rows of pitch ld, c < C
    ld = 4 * C
    w = M.rnd(g, C, s=C ** -0.5, Cr=Cr)
    gh0 = M.rnd(g, nl, ld)
    gh = gh0.cuda()
    call(shim, "add_row", ST, n, C, ld, w.cuda(), 1.3, gh, c["gid"].cuda(), wd)
    sync()
    sc = torch.full((n, 1), 1.3, dtype=torch.float64)
    if wv is not None:
        sc = sc * wv.double()[c["gid"][:n].long()][:, None]
    add = sc * w.double()[None, :]
    check("add_row gh", "readout", gh[:n, :C], M.plus(gh0[:n, :C], add, 2 * add.abs()), what)
    same("add_row other columns", gh[:n, C:], gh0[:n, C:], what)
    same("add_row halo rows", gh[n:], gh0[n:], what)


# ------------------------------------------------------------------------------------------------ edge final
@pytest.mark.parametrize("wgt", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("atomic", [False, True], ids=["noatom", "atom_vir"])
@pytest.mark.parametrize("zbl,agnesi", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["none", "zbl", "agnesi", "zbl_agnesi"])
def test_edge_final(shim, zbl, agnesi, atomic, wgt):
    core = M.core_params(zbl, agnesi)
    for k, c in enumerate(graph_cases(500 + 4 * zbl + 2 * agnesi)):
        nb, nsh = (8, 16) if k != 1 else (64, 9)
        g, E, N = c["g"], c["E"], c["N"]
        d = dev(c)
        g_eb = M.rnd(g, E, 64, s=0.5)
        gY = M.rnd(g, E, 16, s=0.5)
        F0, v0, av0 = M.rnd(g, N, 3), M.rnd(g, 9).double(), M.rnd(g, N, 12)
        F, vir = F0.cuda(), v0.cuda()
        av = av0.cuda() if atomic else None
        wv = (0.5 + torch.rand(N, generator=g)) if wgt else None
        call(shim, "edge_final", ST, M.ctypes.c_int64(E), nsh, d["e_src"], d["e_dst"], d["e_vec"], d["gid"], d["type"],
             *radial_args(nb), *core_args(core), g_eb.cuda(), gY.cuda(), F, vir, av, None if wv is None else wv.cuda())
        sync()
        r = M.edge_final_ref(c, nb, nsh, core, g_eb, gY, F0, v0, av0 if atomic else None, wv)
        what = f"E={E} nb={nb} nsh={nsh}"
        check("edge_final forces", "edge_final", F, r["forces"], what)
        check("edge_final virial", "edge_final", vir, r["virial"], what)
        if atomic:
            check("edge_final atom_vir", "edge_final", av[:, :9], M.Mag(r["atom_vir"].x[:, :9], r["atom_vir"].s[:, :9]),
                  what)
            same("atom_vir pitch columns 9..11", av[:, 9:], av0[:, 9:], what)
        hit = torch.zeros(N, dtype=torch.bool)
        hit[c["gid"].long()[c["e_src"].long()]] = True
        hit[c["gid"].long()[c["e_dst"].long()]] = True
        same("forces of atoms without edges", F[~hit.cuda()], F0[~hit], what)
