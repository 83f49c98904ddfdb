"""MACE step times on the H100 engine for the MACE-MP-0-large shape (DESIGN.md §11.3): perturbed Si with random weights,
hidden features 128x0e + 128x1o + 128x2e, two interactions, max_ell 3, correlation 3, r_max 6 A, 8 Bessel functions,
radial MLP 64-64-64 (tests/mace_medium_times.py times the 0e+1o shape).  Prints one JSON line per size: ms/step and
atoms/s on the resident graph and end to end (graph build + evaluation + copies), device memory per atom, kernel
launches per step, the card's name and power limit, and with --profile the kernel shares of one resident step from
torch.profiler.  --parity also evaluates the last size as a 2-partition group on the same device and prints the largest
energy / force / stress differences against 1 partition.  --fit N1 N2 .. evaluates diamond cells of N^3 unit cells in
ascending order and reports the largest that one partition holds (it stops at the first that does not).

    python tests/mace_large_times.py [--sizes 12 20] [--steps 10] [--profile] [--parity] [--fit 23 24 25]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.mace_l2_ref import make_mace_l2  # noqa: E402
from tests.mace_medium_times import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[12, 20])  # 13 824 and 64 000 atoms
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--parity", action="store_true")
    ap.add_argument("--fit", type=int, nargs="*", default=[])
    a = ap.parse_args()
    m = make_mace_l2(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
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
        launches = eng.counts()["launches"]  # kernel launches of the last evaluation
        eng.compute_resident(reps=3)  # warm-up
        t0 = time.perf_counter()
        eng.compute_resident(reps=a.steps)
        resident = (time.perf_counter() - t0) / a.steps * 1e3
        t0 = time.perf_counter()
        for _ in range(a.steps):
            d.evaluate(atoms)
        e2e = (time.perf_counter() - t0) / a.steps * 1e3
        out = {"natoms": len(atoms), "edges": eng.counts()["n_edges"], "card": card(), "launches_per_step": launches,
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
            out["kernel_shares"] = {k[:60]: round(v / s, 4) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:14]}
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
    best = None
    for n in a.fit:
        atoms = si_diamond(n, seed=1)
        d = None
        try:
            d = ScaleShiftMACE_Dist.from_existing(m)
            d.enable_distributed_mode([0])
            d.evaluate(atoms)
            best = len(atoms)
        except Exception as ex:  # the engine reports a failed allocation as an error; nothing ran on the device
            print(json.dumps({"fit_stopped_at": len(atoms), "error": str(ex)[:200]}), flush=True)
            break
        finally:
            if d is not None and d.__dict__.get("_engine") is not None:
                d._engine.close()
            del d
            torch.cuda.empty_cache()
    if a.fit:
        print(json.dumps({"largest_cell_one_partition": best, "card": card()}), flush=True)


if __name__ == "__main__":
    main()
