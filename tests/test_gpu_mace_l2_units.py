"""The MACE launchers for 0e+1o+2e node features on their own (launch_mace_msg_l2 / _bwd, launch_mace_symc_l2 / _bwd,
launch_mace_elem_mix_rows with 9 components), called through tests/kernel_shim_l2.cu on the synthetic graphs of
tests/mace_units_ref.py, against the float64 restatements of tests/mace_l2_units_ref.py.  Every element must satisfy
|out - ref| <= tol * scale; rows, planes and columns a launch must not write keep their sentinels or prefills bit for
bit.  Cases: partial blocks, E = 1 and 257, n_own = 0 and E = 0, a 300-edge row, halo sources, a self-image edge,
C = 32, 96 and 128 at pitches 64 and 128, max_ell 2 and 3, correlation 1..3."""
import pytest
import torch

from tests import kernel_units_ref as KU
from tests import mace_l2_units_ref as L
from tests import mace_units_ref as M
from tests.mace_units_ref import ST, call

pytestmark = pytest.mark.gpu
ERRS = {}
CH = [(32, 64), (96, 128), (128, 128)]  # (model channels, row pitch)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = KU.Shim(L.build_shim_l2(tmp_path_factory.mktemp("kernel_shim_l2")))
    yield s
    for k in sorted(ERRS):
        print(f"mace-l2-units max |out - ref| / scale  {k:<26s} {ERRS[k]:.3e}")


def check(key, tol, out, ref, what=""):
    KU.check(ERRS, key, L.TOL[tol], out, ref, what)


def same(name, out, before, what=""):
    o, b = out.detach().cpu().contiguous(), before.detach().cpu().contiguous()
    assert torch.equal(o.view(-1).view(torch.int32), b.view(-1).view(torch.int32)), f"{name} {what} changed"


def dev(c):
    return {k: v.cuda() for k, v in c.items() if isinstance(v, torch.Tensor)}


GRAPHS = {"standard": lambda s: M.gen_graph(37, s, empty=3, heavy=300), "E1": lambda s: M.gen_graph(5, s, E=1),
          "E257": lambda s: M.gen_graph(29, s, E=257)}


@pytest.mark.parametrize("graph", list(GRAPHS))
@pytest.mark.parametrize("Cr,C", CH)
@pytest.mark.parametrize("max_ell", [2, 3])
def test_msg_l2_and_reverse(shim, max_ell, Cr, C, graph):
    c = GRAPHS[graph](50 + max_ell + C)
    paths, per, base, nslots = L.l2_layout(max_ell)
    NP, nsh, n, nl, E = len(paths), (max_ell + 1) ** 2, c["n_own"], c["n_loc"], c["E"]
    g = torch.Generator().manual_seed(500 + max_ell + C)
    R = M.rnd(g, E, NP, C, Cr=Cr).reshape(E, NP * C)
    Y = M.sh(M.d64(c["e_vec"][:, :3]), 16).float() if E else torch.zeros(0, 16)
    Y[:, nsh:] = torch.randn(E, 16 - nsh, generator=g)  # columns past nsh are never read
    u = M.rnd(g, nl, 9, C, Cr=Cr).reshape(nl, 9 * C)
    d = dev(c)
    Am = M.sentinel(nslots * n * C + 64)
    call(shim, "msg_l2", 0, ST, max_ell, n, C, d["row_ptr"], d["e_src"], R.cuda(), Y.cuda(), u.cuda(), Am, None, None,
         None)
    torch.cuda.synchronize()
    what = f"max_ell={max_ell} C={Cr}/{C} {graph}"
    check("msg_l2 Am", "msg_l2", Am[: nslots * n * C], M.multilinear(L.msg_l2_fn(c, C, max_ell), dict(R=R, Y=Y, u=u)),
          what)
    assert bool((Am[nslots * n * C:] == M.SENTINEL).all()), f"Am written past its slots {what}"
    nb_ = max(n - 2, 1)  # reverse on the first rows: gR over R for their edges only
    cb = M.restrict(c, nb_)
    Eb = cb["E"]
    gAm = M.rnd(g, nslots, nb_, C)
    gAm.view(-1, C)[:, Cr:] = 0.0
    Rb = R.clone().cuda()
    gY0, gu0 = M.rnd(g, E, 16), M.rnd(g, nl, 9 * C)
    gY, gu = gY0.cuda(), gu0.cuda()
    call(shim, "msg_l2", 1, ST, max_ell, nb_, C, d["row_ptr"], d["e_src"], Rb, Y.cuda(), u.cuda(), None, gAm.cuda(), gY,
         gu)
    torch.cuda.synchronize()
    r = M.multilinear(L.msg_l2_fn(cb, C, max_ell), dict(R=R[:Eb], Y=Y[:Eb], u=u), g=gAm.reshape(-1),
                      wrt=("R", "Y", "u"))
    check("msg_l2_bwd gR (over R)", "msg_l2_bwd", Rb[:Eb], r["R"], what)
    same("R of edges outside the launch", Rb[Eb:], R[Eb:], what)
    check("msg_l2_bwd gY", "msg_l2_bwd", gY[:Eb, 1:nsh], M.plus(gY0[:Eb, 1:nsh], r["Y"][:, 1:nsh]), what)
    same("gY column 0", gY[:, 0], gY0[:, 0], what)
    same("gY columns past nsh", gY[:, nsh:], gY0[:, nsh:], what)
    same("gY of edges outside the launch", gY[Eb:], gY0[Eb:], what)
    check("msg_l2_bwd gu", "msg_l2_bwd", gu, M.plus(gu0, r["u"]), what)


def test_l2_launchers_do_nothing_at_zero(shim):
    """n_own = 0 and E = 0: nothing launched, nothing touched"""
    c = M.gen_graph(0, 5, n_halo=4)
    d = dev(c)
    A = M.sentinel(71, 4, 128)
    call(shim, "msg_l2", 0, ST, 3, 0, 128, d["row_ptr"], d["e_src"], A, A, A, A, None, None, None)
    call(shim, "msg_l2", 1, ST, 3, 0, 128, d["row_ptr"], d["e_src"], A, A, A, None, A, A, A)
    t = torch.zeros(1, 3, dtype=torch.int32).cuda()
    call(shim, "symc_l2", 0, ST, 0, 128, 16, 1, d["type"], A, t, 1, A, None, A)
    call(shim, "symc_l2", 1, ST, 0, 128, 16, 1, d["type"], A, t, 1, A, A, A)
    call(shim, "elem_mix_rows", ST, 0, 128, 9, 9 * 128, 9 * 128, d["type"], A, A, A, 0)
    torch.cuda.synchronize()
    assert bool((A == M.SENTINEL).all())


def test_msg_l2_rejects_max_ell_1(shim):
    c = M.gen_graph(3, 5)
    d = dev(c)
    A = M.sentinel(64)
    with pytest.raises(RuntimeError, match="max_ell"):
        call(shim, "msg_l2", 0, ST, 1, 3, 64, d["row_ptr"], d["e_src"], A, A, A, A, None, None, None)


@pytest.mark.parametrize("accum", [False, True], ids=["set", "accum"])
@pytest.mark.parametrize("Cr,C", CH)
def test_elem_mix_rows_9(shim, accum, Cr, C):
    c = M.gen_graph(37, 80 + C)
    g, n = c["g"], c["n_own"]
    ldi, ldo = 9 * C + 64, 9 * C
    W = M.rnd(g, len(M.ELEMS), 3, C, C, s=C ** -0.5, Cr=Cr)
    W[..., Cr:, :] = 0.0
    x = M.rnd(g, n, ldi)
    x[:, : 9 * C].unflatten(1, (9, C))[..., Cr:] = 0.0
    out0 = M.rnd(g, n + 2, ldo)
    out = out0.cuda()
    call(shim, "elem_mix_rows", ST, n, C, 9, ldi, ldo, c["type"].cuda(), W.cuda(), x.cuda(), out, int(accum))
    torch.cuda.synchronize()
    r = M.multilinear(L.elem_mix_rows9_fn(c, n, C, ldi), dict(W=W, x=x))
    if accum:
        r = M.plus(out0[:n], r.x, r.s)
    check("elem_mix_rows (9) out", "elem_mix", out[:n], r, f"accum={accum} C={Cr}/{C}")
    same("elem_mix_rows (9) rows past n", out[n:], out0[n:])


@pytest.mark.parametrize("corr", [1, 2, 3])
@pytest.mark.parametrize("max_ell", [2, 3])
def test_symc_l2(shim, max_ell, corr):
    Cr, C = CH[(max_ell + corr) % 3]
    seed = 600 + 10 * max_ell + corr
    c = M.gen_graph(37, seed)
    g, n, nsh = c["g"], c["n_own"], (max_ell + 1) ** 2
    mods = L.make_contraction_l2(max_ell, corr, Cr, seed)
    terms = L.build_terms_l2(shim, mods, nsh)
    w, _ = M.stack_weights(mods, C)
    Ktot = w.shape[1]
    A = M.rnd(g, nsh, n, C, s=0.7, Cr=Cr)
    B = M.sentinel(9 * n * C + 64)
    t = c["type"].cuda()
    call(shim, "symc_l2", 0, ST, n, C, nsh, Ktot, t, A.cuda(), terms.cuda(), len(terms), w.cuda(), None, B)
    torch.cuda.synchronize()
    f = L.symc_l2_fn(mods, c, n, C, nsh)
    what = f"max_ell={max_ell} corr={corr} C={Cr}/{C}"
    check("symc_l2 B", "symc", B[: 9 * n * C], M.multilinear(f, dict(A=A)), what)
    assert bool((B[9 * n * C:] == M.SENTINEL).all()), f"B written past its planes {what}"
    gB = M.rnd(g, 9, n, C, Cr=Cr)
    gA = M.sentinel(16, n, C)
    call(shim, "symc_l2", 1, ST, n, C, nsh, Ktot, t, A.cuda(), terms.cuda(), len(terms), w.cuda(), gB.cuda(), gA)
    torch.cuda.synchronize()
    r = M.multilinear(f, dict(A=A), g=gB.reshape(-1), wrt=("A",))
    check("symc_l2_bwd gA", "symc_bwd", gA[:nsh], M.KU_mag(r["A"], (nsh, n, C)), what)
    assert bool((gA[nsh:] == M.SENTINEL).all()), f"planes k >= nsh of gA written {what}"
