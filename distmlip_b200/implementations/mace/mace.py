"""MACECalculator_Dist -- drop-in for DistMLIP's MACE calculator: `MACECalculator_Dist.from_existing(calc)` takes a
mace `MACECalculator` (anything with `models` or `model`, `r_max`, and optionally `energy_units_to_eV` /
`length_units_to_A`), `enable_distributed_mode(gpus)` moves every model of it onto the engine, and `calculate(atoms)`
fills the ASE results.  With `calc_heat_flux=True` (not in mace) every calculation also reads the velocities and masses
of `atoms` and sets `heat_flux` and `heat_flux_potential`, as PESCalculator_Dist does (DESIGN.md §10)."""
from __future__ import annotations

import numpy as np

from distmlip_b200.implementations.matgl.ase import _Calculator, _all_changes, _voigt6

from .models import ScaleShiftMACE_Dist

GPA_PER_EV_A3 = 160.21766208


class MACECalculator_Dist(_Calculator):
    """ASE calculator for one mace model, or a committee of them, on the sm_90a engine."""

    implemented_properties = ("energy", "free_energy", "node_energy", "forces", "stress")

    @classmethod
    def from_existing(cls, calc, calc_heat_flux=False, heat_flux_reach=None):
        """calc_heat_flux and heat_flux_reach (Angstrom, None: each model's receptive field) may be switched between
        calculations"""
        models = list(getattr(calc, "models", None) or [getattr(calc, "model")])
        new = cls()
        new.models = [ScaleShiftMACE_Dist.from_existing(m) for m in models]
        new.num_models = len(new.models)
        new.r_max = float(getattr(calc, "r_max", float(models[0].r_max)))
        new.energy_units_to_eV = float(getattr(calc, "energy_units_to_eV", 1.0))
        new.length_units_to_A = float(getattr(calc, "length_units_to_A", 1.0))
        new.dist_enabled = False
        new.heat_flux_reach = heat_flux_reach
        new.calc_heat_flux = calc_heat_flux
        return new

    @property
    def calc_heat_flux(self):
        return self._calc_heat_flux

    @calc_heat_flux.setter
    def calc_heat_flux(self, on):
        """the flux properties are advertised only while the flux is on"""
        self._calc_heat_flux = bool(on)
        props = tuple(MACECalculator_Dist.implemented_properties)
        if self.num_models > 1:
            props += ("energies", "energy_var", "forces_comm", "stress_var")
        if self._calc_heat_flux:
            props += ("heat_flux", "heat_flux_potential")
        self.implemented_properties = props

    def enable_distributed_mode(self, gpus, balance=False):
        """`balance`: work-balanced slab walls for every model (ScaleShiftMACE_Dist.enable_distributed_mode)"""
        for m in self.models:
            m.enable_distributed_mode(gpus, balance)
        self.dist_enabled = True

    def calculate(self, atoms=None, properties=None, system_changes=None):
        if not self.dist_enabled:
            raise RuntimeError("call enable_distributed_mode(gpus) first")
        super().calculate(atoms, properties, system_changes or _all_changes)
        eu, lu = self.energy_units_to_eV, self.length_units_to_A
        v = np.asarray(atoms.get_velocities(), dtype=np.float64) if self.calc_heat_flux else None
        E, F, S, NE, JP, JC = [], [], [], [], [], []
        for m in self.models:
            if v is not None:
                e, f, s, ae, _, (jp, jc) = m.evaluate_heat_flux(atoms, v, reach=self.heat_flux_reach, atomic=True)
                JP.append(jp * eu)
                JC.append(jc * eu)
            else:
                e, f, s, ae, _ = m.evaluate(atoms, forces=True, stress=True, atomic=True)
            E.append(e * eu)
            F.append(np.asarray(f, dtype=np.float64) * eu / lu)
            S.append(np.asarray(s, dtype=np.float64) / GPA_PER_EV_A3 * eu / lu ** 3)
            NE.append((ae - m._e0[m._species_of(atoms)]) * eu)
        E, F, S, NE = np.array(E), np.stack(F), np.stack(S), np.stack(NE)
        self.results = {
            "energy": float(E.mean()),
            "free_energy": float(E.mean()),
            "node_energy": NE.mean(axis=0),
            "forces": F.mean(axis=0),
            "stress": _voigt6(S.mean(axis=0)),
        }
        if self.num_models > 1:
            self.results["energies"] = E
            self.results["energy_var"] = float(E.var())
            self.results["forces_comm"] = F
            self.results["stress_var"] = _voigt6(S.var(axis=0))
        if v is not None:
            # J = sum_i (eps_i + 1/2 m_i v_i^2) v_i + J_pot (eV * Angstrom / ASE time unit, not divided by the volume)
            j_pot = np.mean(JP, axis=0)
            kin = 0.5 * np.asarray(atoms.get_masses(), dtype=np.float64) * np.einsum("ij,ij->i", v, v)
            self.results["heat_flux"] = np.mean(JC, axis=0) + kin @ v + j_pot
            self.results["heat_flux_potential"] = j_pot
