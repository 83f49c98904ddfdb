"""The TensorNet kernel-unit tests (tests/test_gpu_tn_units.py) without a GPU: the shim builds with the TensorNet
entry points; the kernels' hand-derived reverses, restated in float64, equal autograd of the 3x3 restatement; every
scale bounds its value, and a float32 evaluation of the Gaussian basis and the row GEMM stays within tolerance; and the
tolerances are sharp: on inputs built as the GPU tests build them, every float64 mutant (what a subtly wrong kernel
would compute) exceeds its tolerance by at least MUTANT_MARGIN on some element.  Needs nvcc for the shim, not a GPU.
"""
import os
import re

import pytest
import torch

from tests import kernel_units_ref as KU
from tests import tn_units_ref as T
from tests.test_ptxas_spills import nvcc

RATIOS = {}


def ratio(name, tol, pairs):
    """largest over (mutant value, Mag ref) pairs of max |mut - ref| / scale / tol; recorded and printed"""
    r = max(KU.max_err(mut, ref.x, ref.s) for mut, ref in pairs) / T.TOL[tol]
    RATIOS[name] = min(RATIOS.get(name, float("inf")), r)
    print(f"tn mutant {name:<34s} {r:.3g} x tol")
    return r


def sharp(name, tol, pairs):
    r = ratio(name, tol, pairs)
    assert r >= KU.MUTANT_MARGIN, (name, r)


def test_shim_covers_every_launcher(tmp_path):
    """every launch_tn_* of kernels.cuh has a shim entry point, and the built shim exports each"""
    if nvcc() is None:
        pytest.skip("nvcc not found")
    s = KU.Shim(KU.build_shim(tmp_path))
    here = os.path.dirname(os.path.abspath(__file__))
    decl = open(os.path.join(here, "..", "distmlip_b200", "csrc", "kernels.cuh")).read()
    shim_src = open(os.path.join(here, "kernel_shim.cu")).read()
    for name in set(re.findall(r"void (launch_tn_\w+)\(", decl)):
        assert "b2m::" + name + "(" in shim_src, name
    for entry in set(re.findall(r"int (shim_tn_\w+)\(", shim_src)):
        assert hasattr(s.lib, entry), entry


# ------------------------------------------------------------------------------------------------ hand reverses
def test_hand_reverses_equal_autograd():
    """the kernels' schedule of prod_bwd and update_bwd (float64) against autograd of the 3x3 restatement"""
    g = torch.Generator().manual_seed(3)
    n = 23
    m, y, gp = T.gen_dec(g, n), T.gen_dec(g, n), T.rnd(g, n, 10, 64)
    for so3 in (0, 1):
        r = T.node_ref("prod", n, [m, y], gp, so3=so3)
        gm, gy = T.prod_bwd_hand(T.rows(m, n), T.rows(y, n), T.rows(gp, n), so3)
        assert KU.max_err(T.lay(gm, n), r["gmsg"].x, r["gmsg"].s) < 1e-12
        assert KU.max_err(T.lay(gy, n), r["gY"].x, r["gY"].s) < 1e-12
    d = T.gen_dec(g, n)
    r = T.node_ref("update", n, [m, d], gp)["gdX"]
    assert KU.max_err(T.lay(T.update_bwd_hand(T.rows(d, n), T.rows(gp, n)), n), r.x, r.s) < 1e-12


# ------------------------------------------------------------------------------------------------ scales
def bounded(m, what):
    assert bool((m.s >= m.x.abs() * (1 - 1e-12)).all()), what


def test_scales_bound_values_and_f32():
    g = torch.Generator().manual_seed(4)
    n = 37
    X, Y = T.gen_dec(g, n), T.gen_dec(g, n)
    for op, ins in (("scale", [X]), ("prod", [X, Y]), ("update", [X, Y]), ("invariants", [X])):
        for k, v in T.node_ref(op, n, ins).items():
            bounded(v, f"{op} {k}")
    # where the restatement is the kernel's arithmetic, its float32 evaluation stays within tolerance
    c = T.gen_graph(37, 9, empty=3, heavy=300)
    r = T.edge_geom_ref(c["e_vec"], 20)
    for k, v in r.items():
        bounded(v, k)
    rbf32 = torch.exp(-T.WIDTH * (c["e_vec"][:, 3:4] - T.mu_of(20)[None, :]) ** 2)
    assert KU.max_err(rbf32, r["rbf"].x[:, :20], r["rbf"].s[:, :20]) < T.TOL["edge_geom"]
    E, N = c["E"], c["N"]
    r = T.edge_final_ref(c, 20, T.rnd(g, E, 64), T.rnd(g, E), T.rnd(g, E, 3), T.rnd(g, N, 3), T.rnd(g, 9).double(),
                         T.rnd(g, N, 12))
    for k, v in r.items():
        bounded(v, k)
    A, B = T.rnd(g, 129, 192), T.rnd(g, 192, 64, s=192 ** -0.5)
    ref, _ = T.gemm_ref(A, B)
    assert KU.max_err(A @ B, ref.x, ref.s) < T.TOL["gemm"]


# ------------------------------------------------------------------------------------------------ mutants
def test_gemm_mutants():
    g = torch.Generator().manual_seed(5)
    M, K, N = 127, 192, 128
    A, B, Pre, Cold = T.rnd(g, M, K), T.rnd(g, K, N, s=K ** -0.5), T.rnd(g, M, N, s=2.0), T.rnd(g, M, N)
    ref, _ = T.gemm_ref(A, B, epi=2, Pre=Pre, Cold=Cold, accum=True)
    for mut in ("last_k_chunk_dropped", "rows_64_127_lost", "accum_before_dsilu"):
        m, _ = T.gemm_ref(A, B, epi=2, Pre=Pre, Cold=Cold, accum=True, mut=(mut,))
        sharp(mut + " (gemm)", "gemm", [(m.x, ref)])
    # the channel mix with plane 4 multiplied by B1 instead of B2
    X = T.gen_dec(g, 129).reshape(129, 640)
    B1, B2 = T.rnd(g, 64, 64, s=0.125), T.rnd(g, 64, 64, s=0.125)
    ref, _ = T.gemm_ref(X[:, 256:320], B2)
    sharp("bsel_off_by_one (gemm)", "gemm", [(T.gemm_ref(X[:, 256:320], B1)[0].x, ref)])


def embed_case():
    c = T.gen_graph(37, 50, empty=3, heavy=300)
    g = torch.Generator().manual_seed(52)
    E = c["E"]
    cut = T.edge_geom_ref(c["e_vec"], 20)["cut"].x.float()
    U, V, P = T.rnd(g, T.N_ELEM, 64), T.rnd(g, T.N_ELEM, 64), T.rnd(g, E, 192)
    return c, U, V, P, cut, T.rnd(g, c["n_own"], 10, 64), T.rnd(g, E)


def test_embed_agg_mutants():
    c, U, V, P, cut, gT0, gC0 = embed_case()
    ref = T.embed_agg_ref(c, U, V, P, cut, gT0, gC0)
    for mut in ("uv_swapped", "no_traceless"):
        m = T.embed_agg_ref(c, U, V, P, cut, gT0, gC0, mut=(mut,))
        sharp(mut + " (embed_agg)", "embed_agg", [(m[k].x, ref[k]) for k in ("T0", "nr0")])
    # gvh without its -2/3 v^ tr term, tr = sum_c (g_Sxx + g_Syy + g_Szz) w3 (the S-diagonal rows 4, 7, 9)
    dst, src, ty = c["e_dst"].long(), c["e_src"].long(), c["type"].long()
    vn = T.d64(c["e_vec"][:, :3]) / T.d64(c["e_vec"][:, 3:4])
    w3 = T.d64(P)[:, 128:] * T.d64(cut)[:, None] * (T.d64(U)[ty[src]] + T.d64(V)[ty[dst]])
    gS = T.d64(gT0)[dst]
    tr = ((gS[:, 4] + gS[:, 7] + gS[:, 9]) * w3).sum(1)
    sharp("gvh_no_trace_term (embed_agg_bwd)", "embed_agg_bwd",
          [(ref["gvh"].x + (2.0 / 3.0) * vn * tr[:, None], ref["gvh"])])


def test_layernorm_mutant():
    g = torch.Generator().manual_seed(6)
    x = T.rnd(g, 45, 192, s=2.0)
    gamma, beta, gy = 1 + 0.3 * T.rnd(g, 192), T.rnd(g, 192, s=0.5), T.rnd(g, 45, 192)
    ref = T.layernorm_ref(x, gamma, beta, gy)["gx"]
    m = T.layernorm_ref(x, gamma, beta, gy, mut=("no_xhat_term",))["gx"]
    sharp("no_xhat_term (layernorm_bwd)", "layernorm_bwd", [(m.x, ref)])


def test_node_mutants():
    g = torch.Generator().manual_seed(7)
    n = 37
    X, Y, G = T.gen_dec(g, n), T.gen_dec(g, n), T.rnd(g, n, 10, 64)
    proj = lambda t: T.lay(T.proj(T.rows(t, n)), n)  # noqa: E731
    ref = T.node_ref("scale", n, [X], G)["gX"]
    m = T.node_ref("scale", n, [X], G, mut=("nw_offdiag_1",))["gX"]
    sharp("nw_offdiag_1 (scale_bwd)", "node_bwd", [(proj(m.x), ref)])
    ref = T.node_ref("invariants", n, [X])["inv"]
    m = T.node_ref("invariants", n, [X], mut=("nw_offdiag_1",))["inv"]
    sharp("nw_offdiag_1 (invariants)", "node", [(m.x, ref)])
    s2p = T.rnd(g, n, 192, s=2.0)
    ref = T.node_ref("embed_out", n, [X, s2p])["X0"]
    m = T.node_ref("embed_out", n, [X, s2p], mut=("s2p_blocked",))["X0"]
    sharp("s2p_blocked (embed_out)", "node", [(m.x, ref)])
    for so3 in (0, 1):
        r = T.node_ref("prod", n, [X, Y], G, so3=so3)
        muts = ["dec_adj_no_trace"] + (["so3_order_swapped"] if so3 else ["gm_y_not_yt"])
        for mut in muts:
            if mut == "so3_order_swapped":
                m = T.node_ref("prod", n, [X, Y], G, so3=so3, mut=(mut,))
                gm, gy = m["gmsg"].x, m["gY"].x
            else:
                gm, gy = T.prod_bwd_hand(T.rows(X, n), T.rows(Y, n), T.rows(G, n), so3, mut=(mut,))
                gm, gy = T.lay(gm, n), T.lay(gy, n)
            sharp(f"{mut} (prod_bwd so3={so3})", "node_bwd", [(proj(gm), r["gmsg"]), (proj(gy), r["gY"])])
    r = T.node_ref("update", n, [X, Y], G)["gdX"]
    m = T.lay(T.update_bwd_hand(T.rows(Y, n), T.rows(G, n), mut=("d_not_dt",)), n)
    sharp("d_not_dt (update_bwd)", "node_bwd", [(m, r)])


def test_msg_mutants():
    c = T.gen_graph(37, 130, empty=3, heavy=300)
    n, nl, E = c["n_own"], c["n_loc"], c["E"]
    g = torch.Generator().manual_seed(132)
    f3p = T.rnd(g, E, 192, s=2.0)
    cut = T.edge_geom_ref(c["e_vec"], 20)["cut"].x.float()
    Y = T.gen_dec(g, nl)
    ref = T.msg_ref(c, f3p, cut, Y)["msg"]
    sharp("f3p_blocked (msg)", "msg", [(T.msg_ref(c, f3p, cut, Y, mut=("f3p_blocked",))["msg"].x, ref)])
    gmsg, gC0, gY0 = T.rnd(g, n, 10, 64), T.rnd(g, E), T.rnd(g, nl, 10, 64)
    ref = T.msg_ref(c, f3p, cut, Y, gmsg, gC0, gY0)["gY"]
    m = T.msg_ref(c, f3p, cut, Y, gmsg, gC0, gY0, mut=("gy_to_dst",))["gY"]
    sharp("gy_to_dst (msg_bwd)", "msg_bwd", [(m.x, ref)])


def test_readout_mutants():
    c = T.gen_graph(37, 141)
    g, n, N = c["g"], c["n_own"], c["N"]
    W = 64
    hL, hG, wL, wG = T.rnd(g, n, W), T.rnd(g, n, W), T.rnd(g, W, s=W ** -0.5), T.rnd(g, W, s=W ** -0.5)
    er = torch.linspace(-3.0, -1.0, T.N_ELEM, dtype=torch.float64)
    wv = 0.5 + torch.rand(N, generator=g)
    e0 = torch.tensor([0.25], dtype=torch.float64)
    ref = T.readout_final_ref(c, n, W, hL, wL, 0.3, hG, wG, -0.2, er, 1.3, 0.07, wv, e0)
    for mut in ("eref_wrong_element", "wgt_twice"):
        m = T.readout_final_ref(c, n, W, hL, wL, 0.3, hG, wG, -0.2, er, 1.3, 0.07, wv, e0, mut=(mut,))
        sharp(mut + " (readout_final)", "readout", [(m[k].x, ref[k]) for k in ("energy", "atom_e")])
    lout, gout = T.rnd(g, n), 0.02 + 0.96 * torch.rand(n, generator=g)
    preL, preG = T.rnd(g, n, W, s=2.0), T.rnd(g, n, W, s=2.0)
    ref = T.readout_seed_ref(c, n, lout, gout, 1.3, wL, wG, preL, preG, wv)
    for mut in ("silu_p_as_sigma", "no_g1mg", "wgt_twice"):
        m = T.readout_seed_mutant(c, n, lout, gout, 1.3, wL, wG, preL, preG, wv, (mut,))
        sharp(mut + " (readout_seed)", "readout", [(m[k], ref[k]) for k in ("gL", "gG")])


def test_edge_final_mutants():
    c = T.gen_graph(37, 162, empty=3, heavy=300)
    g, E, N = c["g"], c["E"], c["N"]
    g_rbf, gC, gvh = T.rnd(g, E, 64, s=0.5), T.rnd(g, E), T.rnd(g, E, 3)
    F0, v0, av0 = T.rnd(g, N, 3), T.rnd(g, 9).double(), T.rnd(g, N, 12)
    ref = T.edge_final_ref(c, 32, g_rbf, gC, gvh, F0, v0, av0)
    for mut in ("gauss_no_2", "cut_sign", "no_tangential", "vir_transposed", "atom_vir_all_dst"):
        m = T.edge_final_ref(c, 32, g_rbf, gC, gvh, F0, v0, av0, mut=(mut,))
        sharp(mut + " (edge_final)", "edge_final", [(m[k].x, ref[k]) for k in ref])
