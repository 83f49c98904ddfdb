"""Kernel-unit references of the MACE launchers for 0e+1o+2e node features (k_mace_msg_l2 / _bwd, k_mace_symc_eq with
9 output slots, k_mace_elem_mix_rows with 9 components), in the manner of tests/mace_units_ref.py, whose graphs, scales
(`multilinear`: the same operation on |inputs| and |coefficients|) and contraction helpers they reuse.  Conventions
come from tests/mace_l2_ref.py (paths, coupling tensors, the 2e contraction)."""
from __future__ import annotations

import math
import os
import subprocess

import torch

from oracle import mace_ref as MR
from tests import mace_l2_ref as L2
from tests import mace_units_ref as M
from tests.kernel_units_ref import F64, d64

# |out - ref| <= TOL * scale, per element: the tolerances of the 0e+1o launchers they widen (mace_units_ref.TOL), at
# least 10x below every mutant (tests/test_mace_l2_units_cpu.py)
TOL = {"msg_l2": M.TOL["msg_eq"], "msg_l2_bwd": M.TOL["msg_eq_bwd"], "elem_mix": M.TOL["elem_mix"],
       "symc": M.TOL["symc"], "symc_bwd": M.TOL["symc_bwd"]}
LS9 = [0, 1, 1, 1, 2, 2, 2, 2, 2]  # l of each hidden component


def build_shim_l2(outdir):
    """Compile tests/kernel_shim_l2.cu (kernel_shim.cu and the 0e+1o+2e entry points) against the built libb200mlip.so
    into outdir, as kernel_units_ref.build_shim does for kernel_shim.cu; returns the shared object's path."""
    from distmlip_b200 import build

    lib = build.build()
    libdir = os.path.dirname(lib)
    here = os.path.dirname(os.path.abspath(__file__))
    out = os.path.join(str(outdir), "libkernel_shim_l2.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + [
        "-I", build.CSRC, "-I", os.path.join(here, "..", "include"), "-shared", os.path.join(here, "kernel_shim_l2.cu"),
        "-o", out, "-L", libdir, "-l:" + os.path.basename(lib), "-Xlinker", "-rpath," + libdir]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    return out


def l2_layout(max_ell):
    """conv_tp paths with 0e+1o+2e input, per l_out the path indices, each l_out block's slot base, and the slot count"""
    paths = L2.conv_paths(max_ell, 2)
    per = [[p for p, pt in enumerate(paths) if pt[2] == l] for l in range(max_ell + 1)]
    base, b = [], 0
    for l in range(max_ell + 1):
        base.append(b)
        b += (2 * l + 1) * len(per[l])
    return paths, per, base, b


def msg_l2_fn(c, C, max_ell, mut=()):
    """Am (flat, the slot layout of mace_state.cuh with hidden_l = 2) of k_mace_msg_l2 from R [E][NP][C], Y [E][16],
    u [n_loc][9][C].  Mutants: cg_sign_2e (one coefficient of the first path with l_in = 2 negated), drop_path_2 (the
    last path with l_in = 2 left out)"""
    paths, per, base, nslots = l2_layout(max_ell)
    src, dst, n = c["e_src"].long(), c["e_dst"].long(), c["n_own"]
    NP = len(paths)
    first2 = next(p for p, pt in enumerate(paths) if pt[0] == 2)
    last2 = max(p for p, pt in enumerate(paths) if pt[0] == 2)

    def cg_of(p, absolute):
        li, ls, lo = paths[p]
        cg = L2.make_cg(li, ls, lo).clone() * math.sqrt(2 * lo + 1)
        if "cg_sign_2e" in mut and p == first2:
            i = tuple(int(a) for a in torch.nonzero(cg.abs() > 1e-6)[0])
            cg[i] = -cg[i]
        return cg.abs() if absolute else cg

    def f(absolute, R, Y, u):
        R, u = R.view(-1, NP, C), u.view(-1, 9, C)[src]
        blocks = []
        for lo in range(max_ell + 1):
            cols = []
            for p in per[lo]:
                li, ls, _ = paths[p]
                m = torch.einsum("eic,ej,ijk->ekc", u[:, li * li:(li + 1) ** 2], Y[:, ls * ls:(ls + 1) ** 2],
                                 cg_of(p, absolute)) * R[:, p, None, :]
                if "drop_path_2" in mut and p == last2:
                    m = m * 0.0
                cols.append(torch.zeros(n, 2 * lo + 1, C, dtype=F64).index_add(0, dst, m))
            blocks.append(torch.stack(cols, 2).permute(1, 0, 2, 3).reshape(-1))
        return torch.cat(blocks)
    return f


def elem_mix_rows9_fn(c, n, C, ldi, mut=()):
    """out rows [n][9 C] = in rows (pitch ldi) @ W[type][l(m)] (W [n_elem][3][C][C]).  Mutants: l1_mix_on_2e (the 1o
    block applied to the 2e components), no_2e_skip (the 2e block omitted)"""
    z = c["type"][:n].long()
    ls = torch.tensor([1 if ("l1_mix_on_2e" in mut and l == 2) else l for l in LS9])

    def f(absolute, W, x):
        W = W.view(-1, 3, C, C)[z]
        xr = x.view(n, ldi)[:, :9 * C].view(n, 9, C)
        out = torch.einsum("nkc,nkcd->nkd", xr, W[:, ls])
        if "no_2e_skip" in mut:
            out = torch.cat([out[:, :4], out[:, 4:] * 0.0], 1)
        return out.reshape(n, 9 * C)
    return f


def make_contraction_l2(max_ell, correlation, Cr, seed):
    """contractions.0, .1 (1o) and .2 (2e) of one product block, U and weights rounded to fp32"""
    torch.manual_seed(seed)
    n_elem = len(M.ELEMS)
    mods = [MR.Contraction(max_ell, correlation, n_elem, Cr)] + \
        [L2.ContractionOut(max_ell, correlation, n_elem, Cr, l) for l in (1, 2)]
    with torch.no_grad():
        for m in mods:
            for nu in range(1, correlation + 1):
                U = getattr(m, f"U_matrix_{nu}")
                U.copy_(U.float().double())
                w = m.weight_of(nu)
                w.copy_((w * 4.0).float().double())
    return mods


def build_terms_l2(shim, mods, nsh):
    """the engine's term list for contractions.0, .1 and .2 (mace_sym_terms with ncomp 1, 3, 5)"""
    out, k = [], 0
    for ci, m in enumerate(mods):
        for nu in range(1, m.correlation + 1):
            U = getattr(m, f"U_matrix_{nu}").float()
            K = U.shape[-1]
            out.append(shim.mace_sym_terms(U, nsh, nu, 2 * ci + 1, K, k))
            k += K
    return torch.cat(out)


def symc_l2_fn(mods, c, n, C, nsh, mut=()):
    """B [9][n][C] (slot 0 the 0e output, 1..3 the 1o, 4..8 the 2e components) from A [nsh][n][C] by the contraction
    modules' own forward.  Mutant: slots_4_5_swapped (two 2e outputs exchanged)"""
    z = c["type"][:n].long()
    Cr = mods[0].weight_of(1).shape[2]

    def f(absolute, A):
        Ar = A.view(nsh, n, C).permute(1, 0, 2)[:, :, :Cr]
        outs = []
        for ci, m in enumerate(mods):
            B = M._mutated(m, absolute, mut, ci)(Ar, z)
            outs.append(B[:, None] if ci == 0 else B)
        B = torch.cat(outs, 1)  # [n][9][Cr]
        if "slots_4_5_swapped" in mut:
            B = B[:, [0, 1, 2, 3, 5, 4, 6, 7, 8]]
        B = torch.nn.functional.pad(B, (0, C - Cr))
        return B.permute(1, 0, 2).reshape(-1)
    return f


def terms_fwd9(terms, A, w, z):
    """B [9][n][C] walked over the term list in float64; the slot is the unsigned field of bits 28..31"""
    A, w = d64(A), d64(w)
    n, C = A.shape[1], A.shape[2]
    B = torch.zeros(9, n, C, dtype=F64)
    coef = d64(terms[:, 2].contiguous().view(torch.float32))
    for j in range(len(terms)):
        t = int(terms[j, 0]) & 0xFFFFFFFF
        nu, o = (t >> 24) & 3, t >> 28
        prod = coef[j] * w[z, int(terms[j, 1])]
        for i in [t & 255, (t >> 8) & 255, (t >> 16) & 255][:nu]:
            prod = prod * A[i]
        B[o] += prod
    return B
