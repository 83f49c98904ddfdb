"""MACE step times on the H100 engine for the MACE-MP-0-medium shape (DESIGN.md §11.1): perturbed Si with random weights,
hidden features 128x0e + 128x1o, two interactions, max_ell 3, correlation 3, r_max 6 A, 8 Bessel functions, radial MLP
64-64-64 (tests/mace_times.py times the same model with scalar hidden features).  Prints one JSON line per size: ms/step
and atoms/s on the resident graph and end to end (graph build + evaluation + copies), device memory per atom, and the
kernel shares of one resident step from torch.profiler.  --parity also evaluates the last size as a 2-partition group on
the same device and prints the largest energy / force / stress differences against 1 partition.

    python tests/mace_medium_times.py [--sizes 12 23] [--steps 10] [--profile] [--parity]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.mace_eq_ref import make_mace_eq  # noqa: E402


def card():
    q = "--query-gpu=name,power.limit"
    return subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[12, 23])  # 13 824 and 97 336 atoms
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--parity", action="store_true")
    a = ap.parse_args()
    m = make_mace_eq(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
                  avg_num_neighbors=45.0)
    for n in a.sizes:
        atoms = si_diamond(n, seed=1)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        d = ScaleShiftMACE_Dist.from_existing(m)
        d.enable_distributed_mode([0])
        d.evaluate(atoms)
        eng = d._engine
        free1 = torch.cuda.mem_get_info()[0]
        eng.compute_resident(reps=3)  # warm-up
        t0 = time.perf_counter()
        eng.compute_resident(reps=a.steps)
        resident = (time.perf_counter() - t0) / a.steps * 1e3
        t0 = time.perf_counter()
        for _ in range(a.steps):
            d.evaluate(atoms)
        e2e = (time.perf_counter() - t0) / a.steps * 1e3
        out = {"natoms": len(atoms), "edges": eng.counts()["n_edges"], "card": card(),
               "resident_ms_per_step": resident, "resident_atoms_per_s": len(atoms) / resident * 1e3,
               "end_to_end_ms_per_step": e2e, "end_to_end_atoms_per_s": len(atoms) / e2e * 1e3,
               "device_bytes_per_atom": (free0 - free1) / len(atoms)}
        if a.profile:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                eng.compute_resident(reps=1)
            tot = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA":
                    tot[ev.key] = tot.get(ev.key, 0.0) + ev.device_time_total
            s = sum(tot.values()) or 1.0
            out["kernel_shares"] = {k[:60]: round(v / s, 4) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:12]}
        if a.parity and n == a.sizes[-1]:
            e1, f1, s1, _, _ = d.evaluate(atoms)
            eng.close()
            del d, eng
            d2 = ScaleShiftMACE_Dist.from_existing(m)
            d2.enable_distributed_mode([0, 0])
            e2, f2, s2, _, _ = d2.evaluate(atoms)
            out["parity_2_partitions"] = {"dE_per_atom": abs(e1 - e2) / len(atoms), "dF_max": float(np.abs(f1 - f2).max()),
                                          "dS_max_GPa": float(np.abs(s1 - s2).max())}
            d2._engine.close()
            print(json.dumps(out), flush=True)
            continue
        print(json.dumps(out), flush=True)
        eng.close()
        del d, eng


if __name__ == "__main__":
    main()
