"""Diagnostic (not a test): cost of the heat flux (b2m_set_heat_flux / b2m_compute_heat_flux).  For each workload one
engine on one GPU, one partition, alternates MD-like steps with the flux off (b2m_set_structure of the periodic cell +
b2m_compute) and on (b2m_set_structure of the unfolded cell + b2m_compute_heat_flux); it reports the host time of each
kind of step (both include the graph build), the unfolded atom and edge counts, the device time of the fold and
contraction kernels (torch.profiler over one flux step) and the device memory in use after each state (the engine's
buffers only grow, so this is its peak).  A workload whose unfolded cell does not fit reports the error.  The card's
name and power limit are read in the same run.  Prints a table and a last JSON line.

    python tests/heat_flux_times.py [--workloads chgnet:23,tensornet:30,chgnet:50] [--rounds 3]
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
from tests.atomic_times import card, make_engine  # noqa: E402

HF = re.compile(r"k_hf_")


def used_gb():
    import torch

    free, total = torch.cuda.mem_get_info(0)
    return (total - free) / 2**30


def step(eng, atoms, sp, reach, v):
    eng.set_heat_flux(reach)
    t0 = time.perf_counter()
    eng.set_structure(atoms.get_positions(), atoms.get_cell(), sp, atoms.get_pbc().astype(np.int32))
    if reach > 0:
        eng.compute_heat_flux(v)
    else:
        eng.compute()
    return (time.perf_counter() - t0) * 1e3


def profile_hf(eng, atoms, sp, reach, v):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(eng, atoms, sp, reach, v)
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and HF.search(ev.name):
            k = re.sub(r"\(.*\)$", "", re.sub(r"^void ", "", ev.name).replace("b2m::", ""))
            tot[k] += ev.device_time_total / 1e3
    return dict(sorted(tot.items()))


def run_workload(family, cells, rounds):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, TensorNet_Dist
    from distmlip_b200.random_init import RandomCHGNet, RandomTensorNet

    atoms = si_diamond(cells)
    dm = (CHGNet_Dist.from_existing(RandomCHGNet(seed=0)) if family == "chgnet"
          else TensorNet_Dist.from_existing(RandomTensorNet(seed=0)))
    reach = dm.heat_flux_reach()
    eng = make_engine(family)
    sp = np.zeros(len(atoms), dtype=np.int32)
    v = np.random.default_rng(0).normal(scale=0.05, size=(len(atoms), 3))
    out = dict(family=family, atoms=len(atoms), reach=reach)
    step(eng, atoms, sp, 0.0, v)
    out["edges"] = eng.counts()["n_edges"]
    out["mem_off_gb"] = used_gb()
    try:
        step(eng, atoms, sp, reach, v)
    except Exception as ex:  # noqa: BLE001
        out["error"] = str(ex)[:200]
        eng.close()
        return out
    c = eng.counts()
    out.update(unfolded_atoms=c["n_own"], unfolded_edges=c["n_edges"], mem_on_gb=used_gb())
    ms = {"off": [], "on": []}
    for _ in range(rounds):
        ms["off"].append(step(eng, atoms, sp, 0.0, v))
        ms["on"].append(step(eng, atoms, sp, reach, v))
    out["step_ms_median"] = {k: float(np.median(x)) for k, x in ms.items()}
    out["step_ms_minmax"] = {k: [float(np.min(x)), float(np.max(x))] for k, x in ms.items()}
    out["ratio"] = out["step_ms_median"]["on"] / out["step_ms_median"]["off"]
    out["hf_kernels_ms"] = profile_hf(eng, atoms, sp, reach, v)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="chgnet:23,tensornet:30,chgnet:50",
                    help="family:cells list (C x C x C Si cells: 23 -> 97 336 atoms, 30 -> 216 000, 50 -> 1 M)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    out = []
    for w in args.workloads.split(","):
        family, cells = w.split(":")
        r = run_workload(family, int(cells), args.rounds)
        out.append(r)
        if "error" in r:
            print(f"{family:9s} {r['atoms']:8d} atoms: flux on failed: {r['error']}", flush=True)
            continue
        m = r["step_ms_median"]
        print(f"{family:9s} {r['atoms']:8d} atoms ({r['edges']} edges) -> {r['unfolded_atoms']} unfolded atoms "
              f"({r['unfolded_edges']} edges, reach {r['reach']} A): off {m['off']:.1f} ms, on {m['on']:.1f} ms "
              f"(x{r['ratio']:.2f}); memory {r['mem_off_gb']:.1f} / {r['mem_on_gb']:.1f} GB; "
              + ", ".join(f"{k} {t:.3f} ms" for k, t in r["hf_kernels_ms"].items()), flush=True)
    print(f"card: {info}")
    print(json.dumps({"card": info, "workloads": out}))


if __name__ == "__main__":
    main()
