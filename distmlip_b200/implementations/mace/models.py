"""ScaleShiftMACE_Dist -- a mace `ScaleShiftMACE` with hidden features C x 0e, C x 0e + C x 1o or C x 0e + C x 1o + C x 2e
on the sm_90a engine.

`from_existing` takes any object with mace's attribute tree and `state_dict()` (mace itself need not be importable, so
the model is recognised by structure, not by `isinstance`); `enable_distributed_mode(gpus)` validates the
configuration and creates the engine (b2m_create_mace).  The arithmetic, with every e3nn / mace convention it relies on,
is stated in oracle/mace_ref.py (scalar hidden features), tests/mace_eq_ref.py (0e+1o), tests/mace_l2_ref.py (0e+1o+2e)
and tests/mace_zbl_ref.py (the ZBL pair repulsion and the Agnesi distance transform); the kernels are
csrc/kernels_mace.cu.

Supported configuration (anything else raises NotImplementedError in enable_distributed_mode): ScaleShiftMACE with one
head, hidden_irreps = C x 0e, C x 0e + C x 1o or C x 0e + C x 1o + C x 2e (C a multiple of 32, C <= 128; the shapes of
MACE-MP-0 "small", "medium" and "large"), max_ell <= 3 (>= 1 with 1o, >= 2 with 2e), correlation <= 3, Bessel radial basis
(num_bessel <= 64) times PolynomialCutoff, a FullyConnectedNet radial MLP (hidden widths <= 64),
RealAgnosticResidualInteractionBlock or RealAgnosticInteractionBlock per layer, LinearReadoutBlock on every layer but the
last and NonLinearReadoutBlock (gated SiLU) on the last.  Optional, as in the MACE-MP-0b / MPA-0 / OMAT-0 checkpoints:
`pair_repulsion` (ZBLBasis, keys pair_repulsion_fn.{c, a_exp, a_prefactor, p, covalent_radii}) and an AgnesiTransform
`radial_embedding.distance_transform` (keys q, p, a, covalent_radii).  Other transforms and `apply_cutoff = False` are
refused.  `evaluate_heat_flux` adds the Green-Kubo heat flux of the unfolded cell (DESIGN.md §10) to `evaluate`.
"""
from __future__ import annotations

import numpy as np
import torch

from distmlip_b200 import _lib
from distmlip_b200.implementations.matgl.models._base import EngineBackedModel

# e3nn normalize2mom(SiLU), 1 / sqrt(E[SiLU(z)^2]) for z ~ N(0, 1): used when the model does not carry its own constant
SILU_2MOM = 1.6765324703310909

_RESIDUAL = "RealAgnosticResidualInteractionBlock"
_PLAIN = "RealAgnosticInteractionBlock"
# mace's ZBLBasis and AgnesiTransform state_dict keys (tests/mace_zbl_ref.py); the engine turns each on when they load
_ZBL, _ZBL_KEYS = "pair_repulsion_fn.", {"c", "a_exp", "a_prefactor", "p", "covalent_radii"}
_AGNESI, _AGNESI_KEYS = "radial_embedding.distance_transform.", {"q", "p", "a", "covalent_radii"}


def _parse_irreps(text):
    """'128x0e+128x1o' -> [(128, 0, 'e'), (128, 1, 'o')] (str() of an e3nn Irreps)"""
    out = []
    for part in str(text).replace(" ", "").split("+"):
        mul, ir = part.split("x") if "x" in part else ("1", part)
        out.append((int(mul), int(ir[:-1]), ir[-1]))
    return out


def conv_paths(max_ell, hidden_l):
    """(l_in, l_sh, l_out) of conv_tp in mace's order (tests/mace_eq_ref.py conv_paths, csrc/engine_mace.inl)"""
    paths = [(li, ls, lo) for li in range(hidden_l + 1) for ls in range(max_ell + 1)
             for lo in range(abs(li - ls), min(li + ls, max_ell) + 1) if (li + ls + lo) % 2 == 0]
    return sorted(paths, key=lambda p: p[2])


def _act_cst(module, default=SILU_2MOM):
    act = getattr(module, "act", None) or getattr(module, "non_linearity", None)
    cst = getattr(act, "cst", None)
    return float(cst) if cst is not None else default


class ScaleShiftMACE_Dist(EngineBackedModel):
    """mace ScaleShiftMACE (H100 engine behind DistMLIP's wrapper API)."""

    __version__ = 1

    @classmethod
    def from_existing(cls, model, dtype=torch.float32):
        for name in ("atomic_numbers", "r_max", "interactions", "products", "readouts", "radial_embedding",
                     "node_embedding", "scale_shift", "atomic_energies_fn"):
            if not hasattr(model, name):
                raise TypeError(f"not a mace ScaleShiftMACE: no attribute {name!r}")
        return super().from_existing(model, dtype)

    def heat_flux_reach(self):
        """Receptive-field radius (Angstrom) of an atom's energy, num_interactions * r_max (DESIGN.md §10): h[0] depends
        on the species only, each interaction adds one r_max hop (the readout of layer t sees t + 1 of them), and the
        ZBL pair term and the Agnesi transform act within one edge."""
        return len(self._attr("interactions")) * float(self._attr("r_max"))

    def _describe(self):
        """b2m_mace_desc fields of the model, or NotImplementedError naming the first unsupported option"""
        sd = self._state_dict
        heads = self._attr("heads", None)
        if heads is not None and len(heads) > 1:
            raise NotImplementedError(f"multi-head models are not supported (heads={list(heads)})")
        zbl = {k[len(_ZBL):] for k in sd if k.startswith(_ZBL)}
        if self._attr("pair_repulsion", False) or zbl:
            if not zbl:
                raise NotImplementedError("pair_repulsion = True without pair_repulsion_fn weights is not supported")
            if zbl != _ZBL_KEYS:
                odd = sorted(zbl - _ZBL_KEYS) or sorted(_ZBL_KEYS - zbl)
                raise NotImplementedError(f"pair_repulsion (ZBL): pair_repulsion_fn.{odd[0]} is " +
                                          ("not a ZBLBasis key" if zbl - _ZBL_KEYS else "missing") +
                                          f"; the keys must be {sorted(_ZBL_KEYS)}")
            if sd[_ZBL + "c"].numel() != 4:
                raise NotImplementedError("pair_repulsion (ZBL): pair_repulsion_fn.c must have 4 coefficients")
        rad = self._attr("radial_embedding")
        dt = getattr(rad, "distance_transform", None)
        agn = {k[len(_AGNESI):] for k in sd if k.startswith(_AGNESI)}
        if dt is not None or any(".distance_transform." in k for k in sd):
            if type(dt).__name__ != "AgnesiTransform":
                raise NotImplementedError(f"radial distance_transform {type(dt).__name__} is not supported "
                                          "(only AgnesiTransform)")
            if agn != _AGNESI_KEYS or any(".distance_transform." in k and not k.startswith(_AGNESI) for k in sd):
                raise NotImplementedError(f"radial distance_transform (AgnesiTransform): the keys must be "
                                          f"{sorted(_AGNESI_KEYS)} under {_AGNESI}, not {sorted(agn)}")
        if getattr(rad, "apply_cutoff", True) is False:
            raise NotImplementedError("radial_embedding.apply_cutoff = False (the cutoff after the radial MLP) is not "
                                      "supported")
        if any(k.startswith("radial_embedding.") and k.split(".")[1] not in ("bessel_fn", "cutoff_fn", "distance_transform")
               for k in sd):
            raise NotImplementedError("radial_type other than the Bessel basis is not supported")
        if "radial_embedding.bessel_fn.bessel_weights" not in sd:
            raise NotImplementedError("radial_type other than the Bessel basis is not supported")
        if any("dipole" in k for k in sd):
            raise NotImplementedError("dipole models are not supported")
        z = [int(a) for a in torch.as_tensor(self._attr("atomic_numbers")).tolist()]
        n_elem = len(z)
        C = int(sd["node_embedding.linear.weight"].numel()) // n_elem
        if C % 32 or C > 128:
            raise NotImplementedError(f"hidden_irreps = {C}x0e: C must be a multiple of 32 and at most 128")
        inters = list(self._attr("interactions"))
        T = len(inters)
        if T > 8:
            raise NotImplementedError(f"num_interactions={T}: at most 8")
        pc = "products.0.symmetric_contractions.contractions.0."
        correlation = sum(1 for k in sd if k.startswith(pc + "U_matrix_"))
        if not 1 <= correlation <= 3:
            raise NotImplementedError(f"correlation={correlation}: 1..3 supported")
        if sd[pc + "U_matrix_1"].dim() != 2:
            raise NotImplementedError("equivariant hidden features: contractions.0 (the 0e output) must have U_matrix_1 "
                                      f"[nsh, K], not {list(sd[pc + 'U_matrix_1'].shape)}")
        nsh = int(sd[pc + "U_matrix_1"].shape[0])
        max_ell = int(round(nsh ** 0.5)) - 1
        if (max_ell + 1) ** 2 != nsh or max_ell > 3:
            raise NotImplementedError(f"edge spherical harmonics with {nsh} components: max_ell <= 3 supported")
        hidden_l = self._hidden_l(sd, inters, C, T, n_elem, nsh, max_ell, correlation)
        residual = 0
        avg = [0.0] * 8
        for t, it in enumerate(inters):
            name = type(it).__name__
            if name == _RESIDUAL:
                residual |= 1 << t
            elif name != _PLAIN:
                raise NotImplementedError(f"interactions.{t} is a {name}: only {_RESIDUAL} and {_PLAIN} are supported")
            avg[t] = float(getattr(it, "avg_num_neighbors"))
            hs = [int(sd[k].shape[1]) for k in sorted(
                (k for k in sd if k.startswith(f"interactions.{t}.conv_tp_weights.layer")),
                key=lambda k: int(k.split(".")[3][5:]))]
            if any(h > 64 for h in hs[:-1]):
                raise NotImplementedError(f"radial MLP hidden widths {hs[:-1]}: at most 64")
        readouts = list(self._attr("readouts"))
        for t, ro in enumerate(readouts):
            want = "NonLinearReadoutBlock" if t == T - 1 else "LinearReadoutBlock"
            if type(ro).__name__ != want:
                raise NotImplementedError(f"readouts.{t} is a {type(ro).__name__}: {want} expected")
        if f"readouts.{T - 1}.linear_2.weight" not in sd:
            raise NotImplementedError("the last readout must be a NonLinearReadoutBlock")
        H = int(sd[f"readouts.{T - 1}.linear_2.weight"].numel())
        first_mlp = getattr(inters[0], "conv_tp_weights", None)
        c_act = _act_cst(getattr(first_mlp, "layer0", None)) if first_mlp is not None else SILU_2MOM
        return _lib.MaceDesc(
            n_elem=n_elem, channels=C, max_ell=max_ell, correlation=correlation, num_interactions=T,
            num_bessel=int(sd["radial_embedding.bessel_fn.bessel_weights"].numel()),
            num_polynomial_cutoff=int(round(float(sd["radial_embedding.cutoff_fn.p"]))),
            mlp_hidden=H, residual_mask=residual, hidden_max_l=hidden_l, r_max=float(sd["r_max"]), c_act=c_act,
            avg_num_neighbors=(_lib.C.c_double * 8)(*avg),
            hidden_mul=(_lib.C.c_int32 * 4)(*[C if l <= hidden_l else 0 for l in range(4)]))

    @staticmethod
    def _hidden_l(sd, inters, C, T, n_elem, nsh, max_ell, correlation):
        """0 for hidden_irreps C x 0e, 1 for C x 0e + C x 1o, 2 for C x 0e + C x 1o + C x 2e, from the interactions'
        `hidden_irreps` when they carry it and from the state_dict shapes (contractions.1 / .2, linear_up, the radial
        MLP's n_paths C outputs, interactions.t.linear, products.t.linear, weights_max), each checked against what
        conv_tp's path rule predicts per layer"""
        hl = None
        irreps = getattr(inters[0], "hidden_irreps", None) if inters else None
        if irreps is not None:
            ir = _parse_irreps(irreps)
            if any(l > 2 for _, l, _ in ir):
                raise NotImplementedError(f"hidden_irreps = {irreps}: hidden l = 3 and above (beyond MACE-MP-0 'large', "
                                          "l > 2) are not supported")
            if len({m for m, _, _ in ir}) > 1:
                raise NotImplementedError(f"hidden_irreps = {irreps}: unequal multiplicities across l are not supported")
            shapes = ([(0, "e")], [(0, "e"), (1, "o")], [(0, "e"), (1, "o"), (2, "e")])
            if [(l, p) for _, l, p in ir] not in shapes:
                raise NotImplementedError(f"hidden_irreps = {irreps}: equivariant hidden features other than 0e, 0e+1o "
                                          "and 0e+1o+2e (parity: only 1o and 2e) are not supported")
            hl = len(ir) - 1
        pre = "products.{}.symmetric_contractions.contractions.{}."
        if any(k.startswith("products.") and ".symmetric_contractions.contractions." in k and
               int(k.split(".")[4]) >= 3 for k in sd):
            raise NotImplementedError("equivariant hidden features with hidden l = 3 and above (a fourth contraction, "
                                      "l > 2) are not supported")
        has1 = [any(k.startswith(pre.format(t, 1)) for k in sd) for t in range(T)]
        has2 = [any(k.startswith(pre.format(t, 2)) for k in sd) for t in range(T)]
        for t in range(T):
            u1 = sd.get(pre.format(t, 1) + "U_matrix_1")
            if has1[t] and (u1 is None or u1.dim() != 3):
                raise NotImplementedError(f"equivariant hidden features: products.{t} has contractions.1 without a "
                                          "[3, nsh, K] U_matrix_1 (malformed state_dict)")
            if u1 is not None and u1.shape[0] != 3:
                raise NotImplementedError(f"equivariant hidden features: contractions.1 of products.{t} gives "
                                          f"{u1.shape[0]} components; only 1o (3) is supported (l > 1 is not)")
            u2 = sd.get(pre.format(t, 2) + "U_matrix_1")
            if has2[t] and (u2 is None or u2.dim() != 3 or u2.shape[0] != 5):
                raise NotImplementedError(f"hidden l > 1 (2e): products.{t} has contractions.2 without a [5, nsh, K] "
                                          "U_matrix_1 (only 2e is supported)")
        sd_hl = 2 if any(has2) else 1 if any(has1) else 0
        if (sd_hl if hl is None else hl) == 2 and max_ell < 2:
            raise NotImplementedError(f"hidden l > 1 (2e) needs max_ell >= 2, not max_ell = {max_ell}")
        if hl is None:
            hl = sd_hl
        elif hl != sd_hl and 2 in (hl, sd_hl):
            raise NotImplementedError(f"hidden l > 1 (2e): hidden_irreps = {irreps} but the state_dict has " +
                                      ("no contractions.2" if hl == 2 else "contractions.2") + " (inconsistent model)")
        elif hl == 0 and sd_hl == 1:
            raise NotImplementedError("equivariant hidden features: contractions.1 on a C x 0e model")
        if hl and max_ell < 1:
            raise NotImplementedError("equivariant hidden features need max_ell >= 1")
        what = {0: f"{C}x0e", 1: f"{C}x0e+{C}x1o", 2: f"{C}x0e+{C}x1o+{C}x2e"}[hl]
        l2 = " (hidden l > 1 (2e))" if hl == 2 else ""
        for t in range(T):
            lin, lout = (hl if t > 0 else 0), (hl if t < T - 1 else 0)
            npaths = len(conv_paths(max_ell, lin))
            up = int(sd[f"interactions.{t}.linear_up.weight"].numel())
            if up != (1 + lin) * C * C:
                c1 = round(max(up - C * C, 0) ** 0.5)
                if lin == 1 and c1 * c1 == up - C * C:
                    raise NotImplementedError(f"interactions.{t}.linear_up maps {C}x0e+{c1}x1o: unequal multiplicities "
                                              "across l are not supported")
                raise NotImplementedError(f"interactions.{t}.linear_up has {up} weights, {(1 + lin) * C * C} expected for "
                                          f"hidden_irreps {what}{l2} (equivariant hidden features other than 0e+1o and "
                                          "0e+1o+2e, or unequal multiplicities across l, are not supported)")
            last = max((k for k in sd if k.startswith(f"interactions.{t}.conv_tp_weights.layer")),
                       key=lambda k: int(k.split(".")[3][5:]))
            if int(sd[last].shape[1]) != npaths * C:
                raise NotImplementedError(f"{last} has {int(sd[last].shape[1])} outputs, {npaths} paths x {C} expected"
                                          f"{l2}: equivariant hidden features other than 0e+1o and 0e+1o+2e (parity: "
                                          "only 1o and 2e) are not supported")
            if int(sd[f"interactions.{t}.linear.weight"].numel()) != npaths * C * C:
                raise NotImplementedError(f"interactions.{t}.linear does not match the {npaths} conv_tp paths of "
                                          "0e" + ("+1o" if lin else "") + ("+2e" if lin == 2 else "") +
                                          f" node features{l2}")
            if int(sd[f"products.{t}.linear.weight"].numel()) != (1 + lout) * C * C:
                raise NotImplementedError(f"products.{t}.linear has {int(sd[f'products.{t}.linear.weight'].numel())} "
                                          f"weights, {(1 + lout) * C * C} expected{l2} (unequal multiplicities across l "
                                          "or hidden l > 2 are not supported)")
            if has1[t] != bool(lout):
                raise NotImplementedError(f"equivariant hidden features: products.{t} " +
                                          ("lacks" if lout else "has") + " contractions.1 (only the last layer is 0e)")
            if has2[t] != (lout == 2):
                raise NotImplementedError(f"hidden l > 1 (2e): products.{t} " + ("lacks" if lout == 2 else "has") +
                                          " contractions.2 (only the last layer is 0e)")
            for ci in range(1, lout + 1):
                w = sd.get(pre.format(t, ci) + "weights_max")
                if w is None or w.dim() != 3 or int(w.shape[0]) != n_elem or int(w.shape[2]) != C:
                    raise NotImplementedError(f"products.{t} contractions.{ci} weights_max is not [{n_elem}, K, {C}]" +
                                              (l2 if ci == 2 else "") + " (unequal multiplicities across l are not "
                                              "supported)")
                if sum(1 for k in sd if k.startswith(pre.format(t, ci) + "U_matrix_")) != correlation:
                    raise NotImplementedError(f"products.{t}: contractions.{ci} and contractions.0 differ in correlation")
        return hl

    def enable_distributed_mode(self, gpus, balance=False):
        """mace.py / models.py of the reference: `gpus` are CUDA ordinals, one per partition (a single-process group
        when one process gets several, one rank per GPU under torchrun, a replica for a single GPU).  `balance`: place
        the slab walls so that every partition holds about the same number of edges (DESIGN.md §4.1)."""
        desc = self._describe()
        gpus, rank, world, group = self._process_layout(gpus)
        from distmlip_b200.structures import Z_OF

        sym_of = {z: s for s, z in Z_OF.items()}
        self.__dict__["element_types"] = tuple(sym_of[int(z)] for z in torch.as_tensor(self._attr("atomic_numbers")).tolist())
        self.__dict__["_e0"] = self._state_dict["atomic_energies_fn.atomic_energies"].double().numpy().reshape(-1)
        eng = _lib.Engine(n_elem=desc.n_elem, n_blocks=desc.num_interactions, cutoff=desc.r_max, mace=desc,
                          device=[int(g) for g in gpus] if group else int(gpus[rank]))
        self._attach_engine(eng, gpus, rank, world, group, balance)
        eng.finalize()
        self._engine_finalized = True

    def evaluate(self, atoms, forces=True, stress=True, atomic=False):
        """One evaluation on the engine: (energy, forces [n, 3] eV/A, stress [3, 3] GPa, per-atom energies or None,
        per-atom virials [n, 3, 3] eV or None)."""
        return self._evaluate(atoms, forces, stress, atomic, 0.0, None)

    def evaluate_batch(self, atoms_list, forces=True, stress=True, atomic=False):
        """`evaluate` for many independent structures in one graph build and one evaluation (DESIGN.md §12): a list of
        `evaluate` tuples, one per structure in order.  The model must run on one GPU and one partition."""
        return [(o["energy"], o["forces"], o["stress"], o["atomic_energies"], o["atomic_virials"])
                for o in self._evaluate_batch(atoms_list, forces, stress, atomic)]

    def evaluate_heat_flux(self, atoms, velocities, reach=None, atomic=False):
        """`evaluate` (energy, forces and stress always) plus the heat flux (J_pot [3], J_conv [3]) of velocities
        [n, 3] (DESIGN.md §10), in eV * velocity unit and not divided by the volume: J_conv = sum_i eps_i v_i over the
        per-atom energies eps_i (E0 and shift included), without the kinetic term.  Every other output is the periodic
        one.  reach (Angstrom) defaults to heat_flux_reach() and may not be below it; a later `evaluate` goes back to
        the periodic graph."""
        need = self.heat_flux_reach()
        reach = need if reach is None else float(reach)
        if reach < need:
            raise ValueError(f"heat_flux_reach={reach} is below the model's receptive field {need}")
        v = np.asarray(velocities, dtype=np.float64)
        if v.shape != (len(atoms), 3):
            raise ValueError(f"velocities must be [{len(atoms)}, 3], not {list(v.shape)}")
        return self._evaluate(atoms, True, True, atomic, reach, v)

    def _evaluate(self, atoms, forces, stress, atomic, reach, velocities):
        if not self.__dict__.get("dist_enabled"):
            raise RuntimeError("call enable_distributed_mode(gpus) first")
        eng = self._engine
        if bool(atomic) != self.__dict__.get("_atomic_on", False):
            eng.set_atomic(bool(atomic))
            self._atomic_on = bool(atomic)
        self._set_heat_flux(reach, None)  # before the graph build, which unfolds the cell when reach > 0
        eng.set_structure(np.asarray(atoms.get_positions(wrap=False), dtype=np.float64), np.array(atoms.get_cell()),
                          self._species_of(atoms), np.asarray(atoms.get_pbc(), dtype=np.int32))
        flux = None
        if velocities is not None:
            e, f, s, flux = eng.compute_heat_flux(velocities)
        else:
            e, f, s = eng.compute(forces=forces, stress=stress)
        ae = av = None
        if atomic:
            ae, av = eng.atomic(virials=forces or stress)
        return (e, f, s, ae, av) if flux is None else (e, f, s, ae, av, flux)

    def dist_forward(self, *args, **kwargs):
        raise NotImplementedError("dist_forward over torch graphs does not exist here; use MACECalculator_Dist")
