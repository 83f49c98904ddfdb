"""Cost of the ZBL pair repulsion and the Agnesi distance transform (DESIGN.md §11.2) on the H100 engine: the
MACE-MP-0-medium shape of tests/mace_medium_times.py (perturbed Si, random weights, 128x0e + 128x1o, two interactions,
max_ell 3, correlation 3, r_max 6 A, 8 Bessel functions, radial MLP 64-64-64) with and without ZBL + Agnesi, the same
weights otherwise.  The two models alternate at each size (plain, core, core, plain).  Prints one JSON line per model and
size: ms/step on the resident graph and end to end, and, from a separate torch.profiler pass, the time of the edge
kernels (`k_mace_edge_geom`, `k_mace_zbl`, `k_mace_edge_final`) in one resident step.

    python tests/mace_zbl_times.py [--sizes 12 23] [--steps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.mace_zbl_ref import make_mace_eq  # noqa: E402

EDGE_KERNELS = ("k_mace_edge_geom", "k_mace_zbl", "k_mace_edge_final")


def card():
    q = "--query-gpu=name,power.limit"
    return subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def measure(m, atoms, steps):
    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode([0])
    d.evaluate(atoms)
    eng = d._engine
    eng.compute_resident(reps=3)  # warm-up
    t0 = time.perf_counter()
    eng.compute_resident(reps=steps)
    resident = (time.perf_counter() - t0) / steps * 1e3
    t0 = time.perf_counter()
    for _ in range(steps):
        d.evaluate(atoms)
    e2e = (time.perf_counter() - t0) / steps * 1e3
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.compute_resident(reps=1)
    kern, total = {}, 0.0
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA":
            total += ev.device_time_total
            for k in EDGE_KERNELS:
                if k + "<" in ev.key or k + "(" in ev.key:
                    kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1e3
    out = {"natoms": len(atoms), "edges": eng.counts()["n_edges"], "launches": eng.counts()["launches"],
           "resident_ms_per_step": resident, "end_to_end_ms_per_step": e2e,
           "profiled_step_ms": total / 1e3, "edge_kernel_ms": kern}
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[12, 23])  # 13 824 and 97 336 atoms
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    kw = dict(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
              avg_num_neighbors=45.0)
    models = {"plain": make_mace_eq(**kw), "zbl+agnesi": make_mace_eq(pair_repulsion=True, distance_transform="agnesi", **kw)}
    for n in a.sizes:
        atoms = si_diamond(n, seed=1)
        for name in ("plain", "zbl+agnesi", "zbl+agnesi", "plain"):
            out = measure(models[name], atoms, a.steps)
            print(json.dumps({"model": name, "card": card(), **out}), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
