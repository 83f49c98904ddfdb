"""Kernel-unit tests of the CHGNet hot path: input generators, the shim that calls the shipped launchers, and a plain
float64 restatement of each launcher's operation with a per-element error scale.

Every reference returns, for each output element, its float64 value and a scale: a first-order bound on the rounding
error a correct fp32 kernel can make there, in units of the working precision.  Quantities are carried as `Mag`
(value, scale) pairs: a sum adds scales, a product x.W with exact weights has scale s(x).|W| (so a dot product gets
sum_k |x_k W_k| at least), an elementwise function f has scale |f'(x)| s(x) + |f(x)| (its input's error carried
through, plus its own rounding), a scatter row gets the sum of its contributions' scales plus |prefill|.  The radial
basis be(d) is evaluated from an fp32 distance, so its scale is |be| + |d be/dd| d.  A kernel output passes when
|out - ref| <= tol * scale for every element; rows that receive nothing must equal their prefill bit for bit.

Values of the backward launchers come from torch.autograd of the forward restatement, independent of the
hand-derived reverse the kernels implement; the reverse is written out here only to carry the scales.

`mutants` evaluates float64 variants of each operation that a subtly wrong kernel would compute (one operand
rounded to tf32, the ninth radial function or a bias dropped, rows of a partial tile or of a run lost, a missing
gradient term, swapped activation derivatives); tests/test_kernel_units_cpu.py requires each to exceed the GPU
tolerance by at least 10x on the same inputs.
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess

import torch

from oracle.manual_ref import dsilu, rbf_env, silu

F64 = torch.float64
TM = 128  # rows per tile of the fused kernels and of the row GEMM
SENTINEL = -777.25

# |out - ref| <= TOL * scale, per element.  Set from the H100 run recorded in DESIGN.md section 5 (at least 3x the
# largest error observed) and at least 10x below every mutant (tests/test_kernel_units_cpu.py).
TOL = {"gemm": 8e-6, "atom_fwd": 5e-7, "atom_bwd": 5e-7, "line_fwd": 1e-6, "line_bwd": 2e-6}
MUTANT_MARGIN = 10.0

# CHGNet's radial basis as random_init.py sets it up (bond_expansion: k pi, cutoff 5 A, exponent 5)
FREQ = (math.pi * torch.arange(1, 10, dtype=torch.float32))
RC, P = 5.0, 5


# ------------------------------------------------------------------------------------------------ shim
def build_shim(outdir):
    """Compile tests/kernel_shim.cu against the built libb200mlip.so into outdir; returns the shared object's path."""
    from distmlip_b200 import build

    lib = build.build()
    libdir = os.path.dirname(lib)
    here = os.path.dirname(os.path.abspath(__file__))
    out = os.path.join(str(outdir), "libkernel_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + [
        "-I", build.CSRC, "-I", os.path.join(here, "..", "include"), "-shared", os.path.join(here, "kernel_shim.cu"),
        "-o", out, "-L", libdir, "-l:" + os.path.basename(lib), "-Xlinker", "-rpath," + libdir]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    return out


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Shim:
    """ctypes front of kernel_shim.cu: torch tensors in, b2m::Error raised as RuntimeError."""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)
        self.msg = ctypes.create_string_buffer(1024)
        self.atom_rad = self.lib.shim_atom_rad()

    def _call(self, fn, *args):
        code = fn(*args, self.msg, ctypes.c_int(len(self.msg)))
        if code != 0:
            raise RuntimeError(f"b2m error {code}: {self.msg.value.decode()}")

    # -------- host weight images (engine.cu formatters)
    def canon_split(self, raw, N, K, Kpad=None):
        Kpad = K if Kpad is None else Kpad
        raw = raw.float().contiguous()
        out = torch.empty(2 * N * Kpad, dtype=torch.float32)
        self._call(self.lib.shim_canon_split, _ptr(raw), ctypes.c_int(N), ctypes.c_int(K), ctypes.c_int(Kpad), _ptr(out))
        return out

    def second_layer_can(self, raw128x64, transposed):
        raw = raw128x64.float().contiguous()
        out = torch.empty(16384, dtype=torch.float32)
        self._call(self.lib.shim_second_layer_can, _ptr(raw), ctypes.c_int(int(transposed)), _ptr(out))
        return out

    def line_reverse_can(self, raw128x64):
        raw = raw128x64.float().contiguous()
        out = torch.empty(16384, dtype=torch.float32)
        self._call(self.lib.shim_line_reverse_can, _ptr(raw), _ptr(out))
        return out

    def radial_can(self, M, Wab):
        M, Wab = M.float().contiguous(), Wab.float().contiguous()
        out = torch.empty(self.atom_rad, dtype=torch.float32)
        self._call(self.lib.shim_radial_can, _ptr(M), _ptr(Wab), _ptr(out))
        return out

    # -------- launchers (device tensors)
    def gemm_wg(self, A, lda, Bcan, C, ldc, M, N, K, bias=None, R=None, ldr=0, accum=False, epi=0, Cpre=None, Pre=None,
                ldp=0, num_sms=1, stream=None):
        i = ctypes.c_int
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream
        self._call(self.lib.shim_gemm_wg, ctypes.c_void_p(st), _ptr(A), i(lda),
                   _ptr(Bcan), _ptr(C), i(ldc), i(M), i(N), i(K), _ptr(bias), _ptr(R), i(ldr), i(int(accum)), i(epi),
                   _ptr(Cpre), _ptr(Pre), i(ldp), i(num_sms))

    def atomconv(self, bwd, c, dev, num_sms):
        """c: an atom-conv case (gen_atom) with its device buffers in dev (to_device)."""
        freq = FREQ.contiguous()
        self._call(self.lib.shim_atomconv, ctypes.c_int(int(bwd)),
                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), ctypes.c_int64(c["E"]),
                   _ptr(dev["e_src"]), _ptr(dev["e_dst"]), _ptr(dev["e_bond"]), _ptr(dev["e_vec"]), _ptr(dev["Aproj"]),
                   _ptr(dev["Cproj"]), _ptr(dev.get("Qproj")), _ptr(dev["radial"]), _ptr(dev["W2can"]),
                   _ptr(dev["W2Tcan"]), _ptr(dev["b2"]), _ptr(freq), ctypes.c_float(RC),
                   ctypes.c_float(math.sqrt(2.0 / RC)), ctypes.c_int(P), _ptr(dev.get("agg")), _ptr(dev.get("gagg")),
                   _ptr(dev.get("gA")), _ptr(dev.get("gC")), _ptr(dev.get("gQ")), _ptr(dev.get("gd")),
                   ctypes.c_int(num_sms))

    def line(self, bwd, hidden, c, dev, num_sms):
        self._call(self.lib.shim_line, ctypes.c_int(int(bwd)), ctypes.c_int(int(hidden)),
                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), ctypes.c_int64(c["A"]),
                   _ptr(dev["a_in"]), _ptr(dev["a_out"]), _ptr(dev["a_ctr"]), _ptr(dev["ang"]), _ptr(dev["Ha"]),
                   _ptr(dev["Hb"]), _ptr(dev["Xc"]), _ptr(dev["Wgcan"]), _ptr(dev["WgTcan"]), _ptr(dev.get("W2can")),
                   _ptr(dev.get("W2Tcan")), _ptr(dev.get("b2")), _ptr(dev.get("aggB")), _ptr(dev.get("ang_out")),
                   _ptr(dev.get("gaggB")), _ptr(dev.get("gang")), _ptr(dev.get("gHa")), _ptr(dev.get("gHb")),
                   _ptr(dev.get("gXc")), ctypes.c_int(num_sms))


# ------------------------------------------------------------------------------------------------ scales
class Mag:
    """A float64 value with its error scale (see the module docstring)."""

    def __init__(self, x, s=None):
        self.x = x
        self.s = x.abs() if s is None else s

    def __add__(self, o):
        o = o if isinstance(o, Mag) else Mag(o)
        return Mag(self.x + o.x, self.s + o.s)

    def __mul__(self, o):
        o = o if isinstance(o, Mag) else Mag(o)
        return Mag(self.x * o.x, self.s * o.x.abs() + self.x.abs() * o.s)

    def __getitem__(self, i):
        return Mag(self.x[i], self.s[i])

    def mm(self, W):  # self @ W, W exact
        return Mag(self.x @ W, self.s @ W.abs())

    def sum(self, dim):
        return Mag(self.x.sum(dim), self.s.sum(dim))

    def apply(self, f):  # elementwise f
        x = self.x.detach().requires_grad_(True)
        with torch.enable_grad():
            y = f(x)
            (dy,) = torch.autograd.grad(y.sum(), x)
        y = y.detach()
        return Mag(y, dy.abs() * self.s + y.abs())


def mcat(a, b):
    return Mag(torch.cat([a.x, b.x], 1), torch.cat([a.s, b.s], 1))


def mwhere(c, a, b):
    return Mag(torch.where(c, a.x, b.x), torch.where(c, a.s, b.s))


def scatter(prefill, idx, m):
    """prefill.index_add(idx, m) with the scatter scale; idx entries < 0 are skipped."""
    ok = idx >= 0
    x = prefill.clone().index_add_(0, idx[ok], m.x[ok])
    s = prefill.abs().index_add_(0, idx[ok], m.s[ok])
    return Mag(x, s)


def sigmoid(x):
    return torch.sigmoid(x)


def dsigmoid(x):
    s = torch.sigmoid(x)
    return s * (1 - s)


def radial(d):
    """be(d), d be/dd (k = 0..8) from fp32 distances, as Mags (the basis is evaluated at an fp32 distance)."""
    d = d.to(F64).detach().requires_grad_(True)
    freq = FREQ.to(F64)
    with torch.enable_grad():
        be, dbe = rbf_env(d, freq, RC, P)
        d2 = torch.stack([torch.autograd.grad(dbe[:, k].sum(), d, retain_graph=True)[0] for k in range(9)], 1)
    be, dbe, dd = be.detach(), dbe.detach(), d.detach()[:, None]
    return Mag(be, be.abs() + dbe.abs() * dd), Mag(dbe, dbe.abs() + d2.abs() * dd)


def tf32(x):
    """x rounded to tf32 the way the kernels split operands (round to nearest, ties away, 10 mantissa bits)."""
    u = x.float().contiguous().view(torch.int32).to(torch.int64)
    u = ((u + 0x1000) & 0xFFFFE000)
    u = torch.where(u >= 2**31, u - 2**32, u).to(torch.int32)
    return u.view(torch.float32).to(x.dtype)


def d64(t):
    return None if t is None else t.detach().to(F64)


def max_err(out, ref, scale):
    """max over elements of |out - ref| / scale (inf if out is not finite where ref is)."""
    out = out.detach().cpu().to(F64)
    err = (out - ref).abs() / scale.clamp_min(1e-300)
    err = torch.where(torch.isfinite(out), err, torch.full_like(err, math.inf))
    return float(err.max()) if err.numel() else 0.0


# ------------------------------------------------------------------------------------------------ row GEMM
def gemm_ref(A, W, bias=None, R=None, Cold=None, accum=False, epi=0, Pre=None):
    """C = epi((R | Cold if accum | 0) + A . W^T + bias), W the [N][K] view the kernel's B image holds.  Returns
    (C Mag, Cpre Mag or None).  With R and accum both set, both are added (R, then Cold)."""
    acc = Mag(d64(A)).mm(d64(W).T)
    if bias is not None:
        acc = acc + Mag(d64(bias)[None, :].expand_as(acc.x))
    if R is not None:
        acc = acc + Mag(d64(R))
    if accum:
        acc = acc + Mag(d64(Cold))
    if epi == 1:
        return acc.apply(silu), acc
    if epi == 2:
        return acc * Mag(d64(Pre)).apply(dsilu), None
    return acc, None


def gen_gemm(M, K, N, seed, cross=None):
    """Operands of one row-GEMM launch: A [M][K] and the weight W [N][K] of unit scale, bias, R, the old C and Pre.
    cross = "lo_hi": A > 0 with a tf32 lo part of about 2^-12 |a| against a W that is exactly tf32, so that the lo.hi
    term of the 3xTF32 split carries weight 2^-12 of the scale; "hi_lo": the same with A and W swapped."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    if cross is not None:
        def with_lo(x):
            x = tf32(x.abs() + 0.5)
            return x * (1 + 2.0**-12 + 2.0**-14 * torch.rand(x.shape, generator=g))
        if cross == "lo_hi":
            A, W = with_lo(A), tf32(W.abs())
        else:
            A, W = tf32(A.abs() + 0.5), with_lo(W.abs() / math.sqrt(K))
    return dict(A=A, W=W, bias=torch.randn(N, generator=g), R=torch.randn(M, N, generator=g),
                Cold=torch.randn(M, N, generator=g), Pre=torch.randn(M, N, generator=g) * 2)


# ------------------------------------------------------------------------------------------------ graphs
def _runs(n_keys, n_rows, pattern, g):
    """Ascending keys in [0, n_keys) for n_rows rows.  pattern: "random" (runs of random length), "ones" (every
    key at most once; needs n_rows <= n_keys), "long" (one key takes a run of more than three tiles), "empty" (a third
    of the keys get no rows), "unsorted" (random run lengths, rows shuffled)."""
    if pattern == "ones":
        keys = torch.sort(torch.randperm(n_keys, generator=g)[:n_rows]).values
    elif pattern == "long":
        assert n_rows > 3 * TM + 16
        run = 3 * TM + 16 + int(torch.randint(0, n_rows - 3 * TM - 15, (1,), generator=g))
        rest = torch.randint(0, n_keys - 1, (n_rows - run,), generator=g)
        k0 = n_keys // 2
        rest = rest + (rest >= k0).long()
        keys = torch.sort(torch.cat([torch.full((run,), k0), rest])).values
    else:
        pool = torch.arange(n_keys)
        if pattern == "empty":
            pool = pool[torch.randperm(n_keys, generator=g)[: max(1, (2 * n_keys) // 3)]]
        keys = torch.sort(pool[torch.randint(0, len(pool), (n_rows,), generator=g)]).values
        if pattern == "unsorted":
            keys = keys[torch.randperm(n_rows, generator=g)]
    return keys.int()


def gen_atom(E, layer0, pattern="random", seed=0, near_cut=True):
    """One atom-conv launch meeting the engine's contract: e_dst over n_own owned atoms (ascending unless pattern is
    "unsorted"), e_src over n_loc >= n_own local atoms, every owned bond exactly once as an edge (layer > 0; about
    half the edges), |e_vec.xyz| = e_vec.w <= cutoff (a few within 1e-4 A of it), unit-scale projections and
    weights, random gagg and prefills."""
    g = torch.Generator().manual_seed(seed)
    n_own = E + 3 if pattern == "ones" else max(2, E // 9)
    n_loc = n_own + max(1, n_own // 3)
    dst = _runs(n_own, E, pattern, g)
    src = torch.randint(0, n_loc, (E,), generator=g).int()
    bond = torch.full((E,), -1, dtype=torch.int32)
    B_own = 0
    if not layer0:
        sel = torch.randperm(E, generator=g)[: max(1, E // 2)]
        B_own = len(sel)
        bond[sel] = torch.randperm(B_own, generator=g).int()
    else:  # layer 0 ignores bonds: give it some anyway
        sel = torch.randperm(E, generator=g)[: E // 2]
        bond[sel] = torch.arange(len(sel)).int()
    d = 0.9 + (RC - 0.9) * torch.rand(E, generator=g)
    if near_cut:
        nc = torch.randperm(E, generator=g)[: max(1, E // 16)]
        d[nc] = RC - 1e-4 * torch.rand(len(nc), generator=g)
    u = torch.randn(E, 3, generator=g, dtype=F64)
    u = u / u.norm(dim=1, keepdim=True)
    xyz = (u * d.to(F64)[:, None]).float()
    e_vec = torch.cat([xyz, xyz.to(F64).norm(dim=1, keepdim=True).float()], 1)  # w = |xyz| in fp32
    c = dict(E=E, layer0=layer0, n_own=n_own, n_loc=n_loc, B_own=B_own, e_src=src, e_dst=dst, e_bond=bond, e_vec=e_vec,
             Aproj=torch.randn(n_loc, 128, generator=g) * 0.6, Cproj=torch.randn(n_own, 128, generator=g) * 0.6,
             Qproj=None if layer0 else torch.randn(B_own, 128, generator=g) * 0.6,
             M=torch.randn(128, 9, generator=g) * 0.8, Wab=torch.randn(64, 9, generator=g) * 0.8,
             W2=torch.randn(128, 64, generator=g) / 8.0, b2=torch.randn(128, generator=g) * 0.5,
             agg=torch.randn(n_own, 64, generator=g), gagg=torch.randn(n_own, 64, generator=g),
             gA=torch.randn(n_loc, 128, generator=g), gC=torch.randn(n_own, 128, generator=g),
             gQ=torch.full((max(B_own, 1), 128), SENTINEL), gd=torch.randn(E, generator=g))
    return c


def gen_line(A, hidden, pattern="random", seed=0):
    """One line-graph launch meeting the engine's contract: angles grouped by centre a_ctr, then by out-bond a_out
    (ascending unless pattern is "unsorted"), a_out over the B_own owned bonds, a_in over B_loc > B_own local bonds
    (halo bonds included), ang padded to whole 128-row tiles with NaN rows (as gang), unit-scale inputs and weights."""
    g = torch.Generator().manual_seed(seed)
    B_own = A + 3 if pattern == "ones" else max(2, A // 5)
    B_loc = B_own + max(2, B_own // 2)
    n_loc = max(2, B_own // 3) + 4
    a_out = _runs(B_own, A, pattern, g)
    ctr_of_bond = torch.sort(torch.randint(0, n_loc, (B_own,), generator=g)).values.int()
    a_ctr = ctr_of_bond[a_out.long()]
    a_in = torch.randint(0, B_loc, (A,), generator=g).int()
    if A > 4:  # some a_in into the halo bonds for sure
        a_in[torch.randperm(A, generator=g)[: max(1, A // 4)]] = torch.randint(B_own, B_loc, (max(1, A // 4),), generator=g).int()
    A_pad = (A + TM - 1) // TM * TM
    ang = torch.full((A_pad, 64), float("nan"))
    ang[:A] = torch.randn(A, 64, generator=g)
    gang = torch.full((A_pad, 64), float("nan"))
    gang[:A] = torch.randn(A, 64, generator=g)
    c = dict(A=A, hidden=hidden, B_own=B_own, B_loc=B_loc, n_loc=n_loc, a_in=a_in, a_out=a_out, a_ctr=a_ctr, ang=ang,
             Ha=torch.randn(B_loc, 128, generator=g) * 0.6, Hb=torch.randn(B_own, 128, generator=g) * 0.6,
             Xc=torch.randn(n_loc, 128, generator=g) * 0.6, Wg=torch.randn(128, 64, generator=g) / 8.0,
             W2=torch.randn(128, 64, generator=g) / 8.0 if hidden else None,
             b2=torch.randn(128, generator=g) * 0.5 if hidden else None,
             aggB=torch.randn(B_own, 64, generator=g), gaggB=torch.randn(B_own, 64, generator=g), gang=gang,
             gHa=torch.randn(B_loc, 128, generator=g), gHb=torch.randn(B_own, 128, generator=g),
             gXc=torch.randn(n_loc, 128, generator=g))
    return c


def to_device(c, shim, kind, dev="cuda"):
    """Device buffers of a case, the weight images made by the engine's formatters."""
    out = {k: v.to(dev).contiguous() for k, v in c.items() if isinstance(v, torch.Tensor)}
    if kind == "atom":
        out["radial"] = shim.radial_can(c["M"], c["Wab"]).to(dev)
    else:
        out["Wgcan"] = shim.second_layer_can(c["Wg"], False).to(dev)
        out["WgTcan"] = shim.line_reverse_can(c["Wg"]).to(dev)
    if c.get("W2") is not None:
        out["W2can"] = shim.second_layer_can(c["W2"], False).to(dev)
        out["W2Tcan"] = shim.second_layer_can(c["W2"], True).to(dev)
    return out


# ------------------------------------------------------------------------------------------------ atom conv
def _gates(pre, W2, b2, hidden=True, swap_dsig=False):
    """u, v of the last layer of a GatedMLP and its message silu(u) sigm(v) (plain tensors, autograd-able).
    swap_dsig: sigm(v) with silu'(v) as its derivative (a mutant)."""
    if hidden:
        hid = silu(pre)
        u = hid[:, :64] @ W2[:64].T + b2[:64]
        v = hid[:, 64:] @ W2[64:].T + b2[64:]
    else:
        u, v = pre[:, :64], pre[:, 64:]
    oG = sigmoid(v)
    if swap_dsig:
        oG = oG.detach() + silu(v) - silu(v).detach()
    return silu(u) * oG


def atom_fwd_values(c, Aproj, Cproj, Qproj, d, mut=()):
    """agg contributions m [E][64] of the atom conv (plain float64, autograd-able); mut: mutant names."""
    src, dst, bond = c["e_src"].long(), c["e_dst"].long(), c["e_bond"].long()
    M, Wab, W2, b2 = d64(c["M"]), d64(c["Wab"]), d64(c["W2"]), d64(c["b2"])
    if "tf32_W2" in mut:
        W2 = d64(tf32(c["W2"]))
    if "tf32_radial" in mut:
        M, Wab = d64(tf32(c["M"])), d64(tf32(c["Wab"]))
    if "no_b2_gate" in mut:
        b2 = torch.cat([b2[:64], torch.zeros(64, dtype=F64)])
    be, _ = rbf_env(d, FREQ.to(F64), RC, P)
    if "no_be8" in mut:
        be = torch.cat([be[:, :8], torch.zeros_like(be[:, 8:])], 1)
    beM = be.detach() if "gd_no_M" in mut else be
    T = beM @ M.T
    if Qproj is not None:
        T = torch.where((bond >= 0)[:, None], Qproj[bond.clamp(min=0)], T)
    pre = Aproj[src] + Cproj[dst] + T
    return _gates(pre, W2, b2, swap_dsig="swap_dsig" in mut) * (be @ Wab.T)


def atom_ref(c, rows=None, mut=()):
    """Forward and backward of the atom conv over the edges `rows` (all by default).  Returns {name: (value, scale)}
    for agg (+= on the prefill) and, by autograd, gA, gC (+=; None in layer 0), gQ (= per bond row; None in layer 0)
    and gd (+= on the prefill); scales from the Mag restatement."""
    E = c["E"]
    rows = torch.arange(E) if rows is None else rows
    sub = dict(c)
    for k in ("e_src", "e_dst", "e_bond", "e_vec"):
        sub[k] = c[k][rows]
    Aproj = d64(c["Aproj"]).requires_grad_(True)
    Cproj = d64(c["Cproj"]).requires_grad_(True)
    Qproj = None if c["layer0"] else d64(c["Qproj"]).requires_grad_(True)
    d = d64(sub["e_vec"][:, 3]).requires_grad_(True)
    dst = sub["e_dst"].long()
    gagg = d64(c["gagg"])
    with torch.enable_grad():
        m = atom_fwd_values(sub, Aproj, Cproj, Qproj, d, mut)
        loss = (m * gagg[dst]).sum()
        wrt = [Aproj, Cproj, d] + ([] if Qproj is None else [Qproj])
        grads = torch.autograd.grad(loss, wrt, allow_unused=True)
    m = m.detach()
    agg = d64(c["agg"]).index_add(0, dst, m)
    gd = d64(c["gd"]).clone()
    gd[rows] += grads[2]
    out = dict(agg=agg, gd=gd)
    if not c["layer0"]:
        out["gA"] = d64(c["gA"]) + grads[0]
        out["gC"] = d64(c["gC"]) + grads[1]
        gQ = d64(c["gQ"]).clone()
        hit = torch.zeros(len(gQ), dtype=torch.bool)
        b = sub["e_bond"].long()
        hit[b[b >= 0]] = True
        gQ[hit] = grads[3][hit]
        out["gQ"] = gQ
    return out


def atom_scales(c):
    """Scales of the atom conv's outputs (all edges), from the forward and the reverse written out on Mags; the
    values of this reverse are returned too (they must equal autograd's)."""
    src, dst, bond = c["e_src"].long(), c["e_dst"].long(), c["e_bond"].long()
    M, Wab, W2, b2 = d64(c["M"]), d64(c["Wab"]), d64(c["W2"]), d64(c["b2"])
    be, dbe = radial(c["e_vec"][:, 3])
    T = be.mm(M.T)
    isQ = torch.zeros(c["E"], dtype=torch.bool) if c["layer0"] else bond >= 0
    if not c["layer0"]:
        T = mwhere(isQ[:, None], Mag(d64(c["Qproj"]))[bond.clamp(min=0)], T)
    pre = Mag(d64(c["Aproj"]))[src] + Mag(d64(c["Cproj"]))[dst] + T
    hid = pre.apply(silu)
    u = hid[:, :64].mm(W2[:64].T) + Mag(b2[:64].expand(c["E"], 64))
    v = hid[:, 64:].mm(W2[64:].T) + Mag(b2[64:].expand(c["E"], 64))
    oL, oG, wab = u.apply(silu), v.apply(sigmoid), be.mm(Wab.T)
    msg = oL * oG * wab
    out = dict(agg=scatter(d64(c["agg"]), dst, msg))
    gm = Mag(d64(c["gagg"]))[dst]
    gwab = gm * oL * oG
    gu = gm * oG * wab * u.apply(dsilu)
    gv = gm * oL * wab * v.apply(dsigmoid)
    gpre = mcat(gu.mm(W2[:64]), gv.mm(W2[64:])) * pre.apply(dsilu)
    gdM = (gpre * dbe.mm(M.T)).sum(1)
    gdM = Mag(torch.where(isQ, 0.0, gdM.x), torch.where(isQ, 0.0, gdM.s))
    out["gd"] = Mag(d64(c["gd"])) + (gwab * dbe.mm(Wab.T)).sum(1) + gdM
    if not c["layer0"]:
        out["gA"] = scatter(d64(c["gA"]), src, gpre)
        out["gC"] = scatter(d64(c["gC"]), dst, gpre)
        gQ = Mag(d64(c["gQ"]))
        b = bond[isQ]
        gQ.x[b], gQ.s[b] = gpre.x[isQ], gpre.s[isQ]
        out["gQ"] = gQ
    return out


# ------------------------------------------------------------------------------------------------ line graph
def line_fwd_values(c, Ha, Hb, Xc, ang, mut=()):
    """pre = ((Ha[a_in] + ang.Wg^T) + Hb[a_out]) + Xc[a_ctr] and the message silu(u) sigm(v) (plain float64)."""
    Wg = d64(tf32(c["Wg"])) if "tf32_Wg" in mut else d64(c["Wg"])
    pre = ((Ha[c["a_in"].long()] + ang @ Wg.T) + Hb[c["a_out"].long()]) + Xc[c["a_ctr"].long()]
    if not c["hidden"]:
        return _gates(pre, None, None, hidden=False, swap_dsig="swap_dsig" in mut)
    W2, b2 = d64(c["W2"]), d64(c["b2"])
    if "tf32_W2" in mut:
        W2 = d64(tf32(c["W2"]))
    if "no_b2_gate" in mut:
        b2 = torch.cat([b2[:64], torch.zeros(64, dtype=F64)])
    return _gates(pre, W2, b2, swap_dsig="swap_dsig" in mut)


def line_ref(c, rows=None, mut=()):
    """Forward and backward of the line-graph kernel over the angles `rows` (all by default).  Returns {name: value}:
    hidden: aggB (+=), gang (+= on the prefill); not hidden: ang_out = ang + m, gang = upstream + chain through m;
    both: gHa, gHb, gXc (+=).  Rows of ang_out / gang outside `rows` and past A are None-valued (NaN)."""
    A = c["A"]
    rows = torch.arange(A) if rows is None else rows
    sub = dict(c)
    for k in ("a_in", "a_out", "a_ctr"):
        sub[k] = c[k][rows]
    Ha = d64(c["Ha"]).requires_grad_(True)
    Hb = d64(c["Hb"]).requires_grad_(True)
    Xc = d64(c["Xc"]).requires_grad_(True)
    ang = d64(c["ang"][rows]).requires_grad_(True)
    gang_in = d64(c["gang"])
    with torch.enable_grad():
        m = line_fwd_values(sub, Ha, Hb, Xc, ang, mut)
        if c["hidden"]:
            loss = (m * d64(c["gaggB"])[sub["a_out"].long()]).sum()
        else:
            loss = ((ang + m) * gang_in[rows]).sum()
        gHa, gHb, gXc, gang = torch.autograd.grad(loss, [Ha, Hb, Xc, ang])
    m = m.detach()
    out = dict(gHa=d64(c["gHa"]) + gHa, gHb=d64(c["gHb"]) + gHb, gXc=d64(c["gXc"]) + gXc)
    g_out = gang_in.clone()
    if c["hidden"]:
        out["aggB"] = d64(c["aggB"]).index_add(0, sub["a_out"].long(), m)
        g_out[rows] += gang
    else:
        ao = torch.full_like(gang_in, math.nan)
        ao[rows] = ang.detach() + m
        out["ang_out"] = ao
        g_out[rows] = gang
    out["gang"] = g_out
    return out


def line_scales(c):
    """Scales of the line-graph kernel's outputs from the Mag restatement (values of its reverse included)."""
    A, hidden = c["A"], c["hidden"]
    a_in, a_out, a_ctr = c["a_in"].long(), c["a_out"].long(), c["a_ctr"].long()
    Wg = d64(c["Wg"])
    ang = Mag(d64(c["ang"][:A]))
    pre = ((Mag(d64(c["Ha"]))[a_in] + ang.mm(Wg.T)) + Mag(d64(c["Hb"]))[a_out]) + Mag(d64(c["Xc"]))[a_ctr]
    if hidden:
        W2, b2 = d64(c["W2"]), d64(c["b2"])
        hid = pre.apply(silu)
        u = hid[:, :64].mm(W2[:64].T) + Mag(b2[:64].expand(A, 64))
        v = hid[:, 64:].mm(W2[64:].T) + Mag(b2[64:].expand(A, 64))
    else:
        u, v = pre[:, :64], pre[:, 64:]
    oL, oG = u.apply(silu), v.apply(sigmoid)
    msg = oL * oG
    pad = lambda m: Mag(torch.cat([m.x, torch.full((len(c["ang"]) - A, 64), math.nan, dtype=F64)]),
                        torch.cat([m.s, torch.full((len(c["ang"]) - A, 64), math.nan, dtype=F64)]))
    out = {}
    if hidden:
        out["aggB"] = scatter(d64(c["aggB"]), a_out, msg)
        gm = Mag(d64(c["gaggB"]))[a_out]
    else:
        out["ang_out"] = pad(ang + msg)
        gm = Mag(d64(c["gang"][:A]))
    gu = gm * oG * u.apply(dsilu)
    gv = gm * oL * v.apply(dsigmoid)
    if hidden:
        gpre = mcat(gu.mm(W2[:64]), gv.mm(W2[64:])) * pre.apply(dsilu)
        out["gang"] = pad(Mag(d64(c["gang"][:A])) + gpre.mm(Wg))
    else:
        gpre = mcat(gu, gv)
        out["gang"] = pad(gm + gpre.mm(Wg))
    out["gHa"] = scatter(d64(c["gHa"]), a_in, gpre)
    out["gHb"] = scatter(d64(c["gHb"]), a_out, gpre)
    out["gXc"] = scatter(d64(c["gXc"]), a_ctr, gpre)
    return out


# ------------------------------------------------------------------------------------------------ mutants
def _dropped_rows(n, keys):
    """Rows a kernel would lose by (a) dropping rows 64..127 of a partial last tile, (b) dropping the first part of a
    run that crosses a tile boundary (the rows of that run in the earlier tile).  Empty where the case has neither."""
    out = {}
    last = (n - 1) // TM * TM
    if n % TM > 64:
        out["rows_64_127_of_last_tile"] = torch.arange(last + 64, n)
    k = keys.long()
    for t in range(TM, n, TM):
        if k[t] == k[t - 1]:
            r = t - 1
            while r > 0 and k[r - 1] == k[t]:
                r -= 1
            out["run_head_before_tile_edge"] = torch.arange(r, t)
            break
    return out


def mutants(kind, c):
    """{mutant name: reference outputs {name: value}} for a case (kind: "atom" or "line")."""
    n = c["E"] if kind == "atom" else c["A"]
    ref = atom_ref if kind == "atom" else line_ref
    names = ["tf32_W2", "no_b2_gate", "swap_dsig"]
    if kind == "atom":
        names += ["tf32_radial", "no_be8", "gd_no_M"]
    else:
        names += ["tf32_Wg"]
        if not c["hidden"]:
            names = [x for x in names if x not in ("tf32_W2", "no_b2_gate")]
    out = {name: ref(c, mut=(name,)) for name in names}
    keys = c["e_dst"] if kind == "atom" else c["a_out"]
    for name, drop in _dropped_rows(n, keys).items():
        keep = torch.ones(n, dtype=torch.bool)
        keep[drop] = False
        out[name] = ref(c, rows=torch.nonzero(keep).flatten())
    return out


def gemm_mutant(case, K, N, epi, flags):
    """The row GEMM with the weight rounded to tf32 (one operand of the product in 1xTF32)."""
    bias, R, accum = flags
    W = tf32(case["W"])
    return gemm_ref(case["A"], W, case["bias"] if bias else None, case["R"] if R else None, case["Cold"], accum, epi,
                    case["Pre"])[0].x


def gemm_cross_mutant(case, which):
    """The row GEMM without one 3xTF32 cross term: lo(A).hi(W) ("lo_hi") or hi(A).lo(W) ("hi_lo")."""
    A, W = d64(case["A"]), d64(case["W"])
    Ah, Wh = d64(tf32(case["A"])), d64(tf32(case["W"]))
    full = Ah @ Wh.T + (A - Ah) @ Wh.T + Ah @ (W - Wh).T
    if which == "lo_hi":
        return full - (A - Ah) @ Wh.T
    return full - Ah @ (W - Wh).T
