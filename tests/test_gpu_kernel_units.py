"""Each CHGNet hot-path launcher on its own: the row GEMM (launch_gemm_wg), the atom conv (launch_atomconv_fwd / _bwd)
and the line-graph kernels (launch_line_fwd / _bwd, hidden and not), called through tests/kernel_shim.cu on synthetic
inputs that meet the engine's contract, against the float64 restatement in tests/kernel_units_ref.py.

Every element must satisfy |out - ref| <= tol * scale, the scale being the first-order rounding bound of that element
(kernel_units_ref.py); rows and columns the launch must not touch keep their sentinels or prefills bit for bit.  The
cases aim at the places tile kernels go wrong: partial last tiles (half 1 empty, or partly filled), one to three CTAs
looping over many tiles (odd and even tile counts per CTA: the double-buffer parities), runs of equal keys crossing
tile and CTA boundaries, runs of length 1, keys with no rows, unsorted keys, distances at the cutoff, halo bonds, NaN
padding rows of the angle buffers, strided GEMM operands and the 3xTF32 cross terms.

B2M_KERNEL_UNITS_REPORT=<path> writes the largest normalised error of every launcher output to <path> (JSON).
"""
import json
import os

import pytest
import torch

from tests import kernel_units_ref as R

pytestmark = pytest.mark.gpu
ERRS = {}


def record(key, err):
    ERRS[key] = max(ERRS.get(key, 0.0), err)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    s = R.Shim(R.build_shim(tmp_path_factory.mktemp("kernel_shim")))
    yield s
    path = os.environ.get("B2M_KERNEL_UNITS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({k: ERRS[k] for k in sorted(ERRS)}, f, indent=1)
    for k in sorted(ERRS):
        print(f"kernel-units max |out - ref| / scale  {k:<22s} {ERRS[k]:.3e}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def check(key, tol, out, ref, what=""):
    """out (device) against a Mag ref, every element; records the largest normalised error under key."""
    err = R.max_err(out, ref.x, ref.s)
    record(key, err)
    if err > tol:
        o = out.detach().cpu().double()
        e = (o - ref.x).abs() / ref.s
        e = torch.where(torch.isfinite(o), e, torch.full_like(e, float("inf")))
        idx = torch.nonzero(e > tol)
        rows = sorted(set(idx[:, 0].tolist())) if idx.ndim == 2 else idx.tolist()
        pytest.fail(f"{key} {what}: max err {err:.3e} > tol {tol:.1e}; {len(idx)} elements in rows "
                    f"{rows[:20]} (tiles {sorted(set(r // R.TM for r in rows))[:20]})")


def untouched(name, out, before, rows_hit, what=""):
    """rows of out that no row of the launch maps to equal their prefill bit for bit"""
    free = torch.ones(len(before), dtype=torch.bool)
    free[rows_hit[rows_hit >= 0].long()] = False
    o = out.detach().cpu()
    same = (o[free].view(torch.int32) == before[free].view(torch.int32)).all()
    assert bool(same), f"{name} {what}: rows without contributions changed"


# ------------------------------------------------------------------------------------------------ row GEMM
GEMM_M = [1, 7, 63, 64, 65, 127, 128, 129, 257]
FLAGS = [(b, r, a) for b in (False, True) for r in (False, True) for a in (False, True)]


def run_gemm(shim, case, K, N, epi, flags, num_sms, off):
    """One launch with A, C, Cpre and Pre as strided views (pitch +64 floats, column offset `off`), C rows >= M and
    columns outside the view holding sentinels (or, for the view with accum, the old C).  Returns (C, Cpre) views."""
    bias, R_on, accum = flags
    M = case["A"].shape[0]
    dev = "cuda"
    lda, ldc, ldr, ldp = K + 64, N + 64, N + 32, N + 64
    Abuf = torch.full((M, lda), R.SENTINEL, device=dev)
    Abuf[:, off:off + K] = case["A"].to(dev)
    Cbuf = torch.full((M + 5, ldc), R.SENTINEL, device=dev)
    if accum:
        Cbuf[:M, off:off + N] = case["Cold"].to(dev)
    Pbuf = torch.full((M + 5, ldc), R.SENTINEL, device=dev)
    Rbuf = torch.full((M, ldr), R.SENTINEL, device=dev)
    Rbuf[:, :N] = case["R"].to(dev)
    Prebuf = torch.full((M, ldp), R.SENTINEL, device=dev)
    Prebuf[:, off:off + N] = case["Pre"].to(dev)
    before_C, before_P = Cbuf.clone(), Pbuf.clone()
    Bcan = shim.canon_split(case["W"], N, K).to(dev)
    b = case["bias"].to(dev)
    shim.gemm_wg(Abuf[:, off:], lda, Bcan, Cbuf[:, off:], ldc, M, N, K, bias=b if bias else None,
                 R=Rbuf if R_on else None, ldr=ldr, accum=accum, epi=epi, Cpre=Pbuf[:, off:] if epi == 1 else None,
                 Pre=Prebuf[:, off:] if epi == 2 else None, ldp=ldp, num_sms=num_sms)
    torch.cuda.synchronize()
    outside = torch.ones_like(Cbuf, dtype=torch.bool)
    outside[:M, off:off + N] = False
    assert torch.equal(Cbuf[outside], before_C[outside]), "C written outside rows < M / its N columns"
    assert torch.equal(Pbuf[outside], before_P[outside]), "Cpre written outside rows < M / its N columns"
    if epi != 1:
        assert torch.equal(Pbuf, before_P), "Cpre written without epi 1"
    return Cbuf[:M, off:off + N], Pbuf[:M, off:off + N]


def gemm_check(shim, case, K, N, epi, flags, num_sms, off, what):
    bias, R_on, accum = flags
    C, Cpre = run_gemm(shim, case, K, N, epi, flags, num_sms, off)
    ref, pre = R.gemm_ref(case["A"], case["W"], case["bias"] if bias else None, case["R"] if R_on else None,
                          case["Cold"], accum, epi, case["Pre"])
    check("gemm_wg C", R.TOL["gemm"], C, ref, what)
    if epi == 1:
        check("gemm_wg Cpre", R.TOL["gemm"], Cpre, pre, what)


@pytest.mark.parametrize("epi", [0, 1, 2])
@pytest.mark.parametrize("K,N", [(64, 128), (64, 64), (128, 64)])
def test_gemm_wg_shapes_sizes_flags(shim, K, N, epi):
    for i, M in enumerate(GEMM_M):
        case = R.gen_gemm(M, K, N, seed=1000 * K + 10 * N + epi + M)
        for flags in FLAGS:
            gemm_check(shim, case, K, N, epi, flags, sms(), 64 * (i & 1), f"M={M} flags={flags}")


@pytest.mark.parametrize("num_sms", [1, 3])
@pytest.mark.parametrize("K,N", [(64, 128), (64, 64), (128, 64)])
def test_gemm_wg_persistent_loop(shim, K, N, num_sms):
    M = 128 * (2 * 2 * num_sms + 1) + 37  # more tiles than the grid (two CTAs per SM at most), last one partial
    case = R.gen_gemm(M, K, N, seed=7 + K + N + num_sms)
    for epi in (0, 1, 2):
        gemm_check(shim, case, K, N, epi, (True, False, True), num_sms, 64, f"M={M} epi={epi}")


def test_gemm_wg_split_k_composition(shim):
    """tc_mm's reverse product with K = 192 in three 64-deep chunks into N = 128: bias and R with the first chunk, the
    others accumulate, the last applies SiLU'(Pre)."""
    M, K, N = 301, 192, 128
    case = R.gen_gemm(M, K, N, seed=77)
    dev = "cuda"
    A = case["A"].to(dev)
    C = torch.full((M, N), R.SENTINEL, device=dev)
    Rm, Pre, b = case["R"].to(dev), case["Pre"].to(dev), case["bias"].to(dev)
    for k0 in (0, 64, 128):
        Bcan = shim.canon_split(case["W"][:, k0:k0 + 64].contiguous(), N, 64).to(dev)
        first, last = k0 == 0, k0 == 128
        shim.gemm_wg(A[:, k0:], K, Bcan, C, N, M, N, 64, bias=b if first else None, R=Rm if first else None, ldr=N,
                     accum=not first, epi=2 if last else 0, Pre=Pre if last else None, ldp=N, num_sms=2)
    torch.cuda.synchronize()
    ref, _ = R.gemm_ref(case["A"], case["W"], case["bias"], case["R"], None, False, 2, case["Pre"])
    check("gemm_wg split-K", R.TOL["gemm"], C, ref)


@pytest.mark.parametrize("cross", ["lo_hi", "hi_lo"])
def test_gemm_wg_3xtf32_cross_terms(shim, cross):
    """Operands whose lo part carries 2^-12 of the scale against an exactly-tf32 partner: without the lo.hi (hi.lo)
    term the error would be about 2^-12 of the scale (tests/test_kernel_units_cpu.py)."""
    for K, N in [(64, 128), (64, 64), (128, 64)]:
        case = R.gen_gemm(257, K, N, seed=5, cross=cross)
        gemm_check(shim, case, K, N, 0, (False, False, False), 2, 0, f"{cross} K={K} N={N}")


# ------------------------------------------------------------------------------------------------ atom conv
COUNTS = [1, 63, 64, 65, 127, 128, 129, 2 * 128 + 1, 3 * 128 + 40, 4 * 128 + 64 + 1, 5 * 128 + 127]


def run_atom(shim, c, num_sms, ref, what):
    dev = R.to_device(c, shim, "atom")
    l0 = c["layer0"]
    # forward: agg += m
    shim.atomconv(False, c, dev, num_sms)
    torch.cuda.synchronize()
    check("atomconv_fwd agg", R.TOL["atom_fwd"], dev["agg"], ref["agg"], what)
    untouched("agg", dev["agg"], c["agg"], c["e_dst"], what)
    # backward: gA / gC += (skipped in layer 0: gA null), gQ = (layer > 0), gd +=
    bw = dict(dev)
    for k in ("gC", "gQ", "gd", "gA"):
        bw[k] = c[k].to("cuda").clone()
    if l0:
        bw["gA"] = None
    shim.atomconv(True, c, bw, num_sms)
    torch.cuda.synchronize()
    check("atomconv_bwd gd", R.TOL["atom_bwd"], bw["gd"], ref["gd"], what)
    if l0:
        assert torch.equal(bw["gC"].cpu(), c["gC"]), f"gC written in layer 0 {what}"
        assert torch.equal(bw["gQ"].cpu(), c["gQ"]), f"gQ written in layer 0 {what}"
    else:
        check("atomconv_bwd gA", R.TOL["atom_bwd"], bw["gA"], ref["gA"], what)
        check("atomconv_bwd gC", R.TOL["atom_bwd"], bw["gC"], ref["gC"], what)
        check("atomconv_bwd gQ", R.TOL["atom_bwd"], bw["gQ"][: c["B_own"]], ref["gQ"][: c["B_own"]], what)
        untouched("gA", bw["gA"], c["gA"], c["e_src"], what)
        untouched("gC", bw["gC"], c["gC"], c["e_dst"], what)


def with_autograd_values(values, scales):
    """the reference: values by autograd of the forward restatement, scales from the Mag restatement"""
    return {k: R.Mag(v, scales[k].s) for k, v in values.items()}


def atom_case(E, layer0, pattern, seed):
    c = R.gen_atom(E, layer0, pattern, seed)
    return c, with_autograd_values(R.atom_ref(c), R.atom_scales(c))


@pytest.mark.parametrize("layer0", [True, False], ids=["layer0", "layerN"])
@pytest.mark.parametrize("E", COUNTS)
def test_atomconv_counts(shim, E, layer0):
    c, ref = atom_case(E, layer0, "random", seed=E)
    for num_sms in (1, 2, 3):
        run_atom(shim, c, num_sms, ref, f"E={E} num_sms={num_sms}")


@pytest.mark.parametrize("layer0", [True, False], ids=["layer0", "layerN"])
@pytest.mark.parametrize("pattern", ["long", "ones", "empty", "unsorted"])
def test_atomconv_run_patterns(shim, pattern, layer0):
    E = 6 * 128 + 45
    c, ref = atom_case(E, layer0, pattern, seed=31)
    for num_sms in (1, 2, 3):
        run_atom(shim, c, num_sms, ref, f"{pattern} E={E} num_sms={num_sms}")


def test_atomconv_more_tiles_than_sms(shim):
    E = 2 * 128 * sms() + 77
    c, ref = atom_case(E, False, "random", seed=3)
    run_atom(shim, c, sms(), ref, f"E={E} num_sms={sms()}")


# ------------------------------------------------------------------------------------------------ line graph
def line_ref_mag(c):
    return with_autograd_values(R.line_ref(c), R.line_scales(c))


def run_line(shim, c, num_sms, ref, what):
    A, hidden = c["A"], c["hidden"]
    dev = R.to_device(c, shim, "line")
    if hidden:
        shim.line(False, True, c, dev, num_sms)
        torch.cuda.synchronize()
        check("line_fwd<H> aggB", R.TOL["line_fwd"], dev["aggB"], ref["aggB"], what)
        untouched("aggB", dev["aggB"], c["aggB"], c["a_out"], what)
    else:
        dev["ang_out"] = torch.full_like(dev["ang"], R.SENTINEL)
        shim.line(False, False, c, dev, num_sms)
        torch.cuda.synchronize()
        check("line_fwd<!H> ang_out", R.TOL["line_fwd"], dev["ang_out"][:A], ref["ang_out"][:A], what)
        assert bool((dev["ang_out"][A:] == R.SENTINEL).all()), f"ang_out padding rows written {what}"
    tag = "H" if hidden else "!H"
    shim.line(True, hidden, c, dev, num_sms)
    torch.cuda.synchronize()
    check(f"line_bwd<{tag}> gang", R.TOL["line_bwd"], dev["gang"][:A], ref["gang"][:A], what)
    assert bool(torch.isnan(dev["gang"][A:]).all()), f"gang padding rows touched {what}"
    for k, idx in (("gHa", "a_in"), ("gHb", "a_out"), ("gXc", "a_ctr")):
        check(f"line_bwd<{tag}> {k}", R.TOL["line_bwd"], dev[k], ref[k], what)
        untouched(k, dev[k], c[k], c[idx], what)


@pytest.mark.parametrize("hidden", [True, False], ids=["H", "notH"])
@pytest.mark.parametrize("A", COUNTS)
def test_line_counts(shim, A, hidden):
    c = R.gen_line(A, hidden, "random", seed=A + 1)
    ref = line_ref_mag(c)
    for num_sms in (1, 2, 3):
        run_line(shim, c, num_sms, ref, f"A={A} num_sms={num_sms}")


@pytest.mark.parametrize("hidden", [True, False], ids=["H", "notH"])
@pytest.mark.parametrize("pattern", ["long", "ones", "empty", "unsorted"])
def test_line_run_patterns(shim, pattern, hidden):
    A = 6 * 128 + 45
    c = R.gen_line(A, hidden, pattern, seed=17)
    ref = line_ref_mag(c)
    for num_sms in (1, 2, 3):
        run_line(shim, c, num_sms, ref, f"{pattern} A={A} num_sms={num_sms}")


@pytest.mark.parametrize("hidden", [True, False], ids=["H", "notH"])
def test_line_more_tiles_than_sms(shim, hidden):
    A = 2 * 128 * sms() + 99
    c = R.gen_line(A, hidden, "random", seed=5)
    run_line(shim, c, sms(), line_ref_mag(c), f"A={A} num_sms={sms()}")

