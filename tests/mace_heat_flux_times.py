"""Diagnostic (not a test): cost of the MACE heat flux (ScaleShiftMACE_Dist.evaluate_heat_flux) for the MACE-MP-0
"small" (128x0e, tests/mace_times.py) and "medium" (128x0e + 128x1o, tests/mace_medium_times.py) shapes: perturbed Si,
random weights, two interactions, max_ell 3, correlation 3, r_max 6 A (reach 12 A).  For each workload one engine on one
GPU, one partition, alternates MD-like steps with the flux off (`evaluate`: graph build of the periodic cell and one
evaluation) and on (`evaluate_heat_flux`: graph build of the unfolded cell and the four passes); it reports the host time
of each kind of step, the unfolded atom and edge counts, the launches per evaluation with the flux off, the device time
of the `k_hf_*` kernels (torch.profiler over one flux step) and the device memory in use after each state (the engine's
buffers only grow, so this is its peak).  A workload whose unfolded cell does not fit reports the error.  The card's name
and power limit are read in the same run.  Prints a table and a last JSON line.

    python tests/mace_heat_flux_times.py [--workloads small:23,medium:12,medium:20] [--rounds 3]
"""
import argparse
import json
import os
import re
import sys
import time
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.heat_flux_times import used_gb  # noqa: E402
from tests.mace_zbl_times import card  # noqa: E402

HF = re.compile(r"k_hf_")


def make(shape):
    from oracle.mace_ref import make_mace
    from tests.mace_eq_ref import make_mace_eq

    kw = dict(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
              avg_num_neighbors=45.0)
    return (make_mace_eq if shape == "medium" else make_mace)(**kw)


def step(d, atoms, v, on):
    t0 = time.perf_counter()
    if on:
        d.evaluate_heat_flux(atoms, v)
    else:
        d.evaluate(atoms)
    return (time.perf_counter() - t0) * 1e3


def profile_hf(d, atoms, v):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(d, atoms, v, True)
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and HF.search(ev.name):
            k = re.sub(r"\(.*\)$", "", re.sub(r"^void ", "", ev.name).replace("b2m::", ""))
            tot[k] += ev.device_time_total / 1e3
    return dict(sorted(tot.items()))


def run_workload(shape, cells, rounds):
    import torch

    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist

    atoms = si_diamond(cells, seed=1)
    d = ScaleShiftMACE_Dist.from_existing(make(shape))
    d.enable_distributed_mode([0])
    v = np.random.default_rng(0).normal(scale=0.05, size=(len(atoms), 3))
    out = dict(shape=shape, atoms=len(atoms), reach=d.heat_flux_reach())
    step(d, atoms, v, False)
    c = d._engine.counts()
    out.update(edges=c["n_edges"], launches_off=c["launches"], mem_off_gb=used_gb())
    try:
        step(d, atoms, v, True)
    except Exception as ex:  # noqa: BLE001
        out["error"] = str(ex)[:200]
        d._engine.close()
        torch.cuda.empty_cache()
        return out
    c = d._engine.counts()
    out.update(unfolded_atoms=c["n_own"], unfolded_edges=c["n_edges"], mem_on_gb=used_gb())
    ms = {"off": [], "on": []}
    for _ in range(rounds):
        ms["off"].append(step(d, atoms, v, False))
        ms["on"].append(step(d, atoms, v, True))
    out["step_ms_median"] = {k: float(np.median(x)) for k, x in ms.items()}
    out["step_ms_minmax"] = {k: [float(np.min(x)), float(np.max(x))] for k, x in ms.items()}
    out["ratio"] = out["step_ms_median"]["on"] / out["step_ms_median"]["off"]
    out["unfold_factor"] = out["unfolded_atoms"] / out["atoms"]
    out["hf_kernels_ms"] = profile_hf(d, atoms, v)
    d._engine.close()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="small:23,medium:12,medium:20",
                    help="shape:cells list (C x C x C Si cells: 12 -> 13 824 atoms, 20 -> 64 000, 23 -> 97 336)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    out = []
    for w in args.workloads.split(","):
        shape, cells = w.split(":")
        r = run_workload(shape, int(cells), args.rounds)
        out.append(r)
        if "error" in r:
            print(f"{shape:6s} {r['atoms']:8d} atoms: flux on failed: {r['error']}", flush=True)
            continue
        m = r["step_ms_median"]
        print(f"{shape:6s} {r['atoms']:8d} atoms ({r['edges']} edges, {r['launches_off']} launches) -> "
              f"{r['unfolded_atoms']} unfolded atoms (x{r['unfold_factor']:.2f}, {r['unfolded_edges']} edges, reach "
              f"{r['reach']} A): off {m['off']:.1f} ms, on {m['on']:.1f} ms (x{r['ratio']:.2f}); memory "
              f"{r['mem_off_gb']:.1f} / {r['mem_on_gb']:.1f} GB; "
              + ", ".join(f"{k} {t:.3f} ms" for k, t in r["hf_kernels_ms"].items()), flush=True)
    print(f"card: {info}")
    print(json.dumps({"card": info, "workloads": out}))


if __name__ == "__main__":
    main()
