"""Diagnostic (not a test): cost of per-atom energies and virials (b2m_set_atomic).  For each workload one engine on one
GPU, one partition, runs rounds that alternate the off and on states on the same resident graph; per state it reports
the device time of an energy+forces+stress step (CUDA events, b2m_compute_resident) and, in the on state, the host time
of fetching the per-atom arrays (b2m_get_atomic).  A short torch.profiler pass per state gives the device time of the
final-stage kernels (readout, k_*edge_final, k_halo_bond_final) and of all memsets of a step (the per-atom arrays are
zeroed by two of them).  The card's
name and power limit are read in the same run.  Prints a table and a last JSON line.

    python tests/atomic_times.py [--workloads chgnet:23,chgnet:50,tensornet:30] [--rounds 4] [--steps 5] [--warmup 3]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.structures import si_diamond  # noqa: E402


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:100]}


def make_engine(family):
    from distmlip_b200.implementations.matgl import CHGNet_Dist, TensorNet_Dist
    from distmlip_b200.random_init import RandomCHGNet, RandomTensorNet

    dm = (CHGNet_Dist.from_existing(RandomCHGNet(seed=0)) if family == "chgnet"
          else TensorNet_Dist.from_existing(RandomTensorNet(seed=0)))
    dm.enable_distributed_mode([0])
    dm._finalize(0.0, 1.0, None)
    return dm._engine


FINAL = re.compile(r"rowdot|readout_final|edge_final|halo_bond_final|memset", re.I)


def profile_final(eng, steps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.compute_resident(1)
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and FINAL.search(ev.name):
            k = re.sub(r"^void ", "", ev.name).replace("(anonymous namespace)::", "").replace("b2m::", "")
            k = re.sub(r"\(.*\)$", "", k)
            tot[k] += ev.device_time_total / 1e3 / steps
    return dict(sorted(tot.items()))


def run_workload(family, cells, rounds, steps, warmup):
    atoms = si_diamond(cells)
    eng = make_engine(family)
    eng.set_structure(atoms.get_positions(), atoms.get_cell(), np.zeros(len(atoms), dtype=np.int32),
                      atoms.get_pbc().astype(np.int32))
    dev = {"off": [], "on": []}
    fetch = []
    launches = {}
    for state in ("off", "on"):  # warm both states (the first on-step allocates the per-atom arrays)
        eng.set_atomic(state == "on")
        for _ in range(warmup):
            eng.compute_resident(1)
    for _r in range(rounds):
        for state in ("off", "on"):
            eng.set_atomic(state == "on")
            eng.compute_resident(1)
            for _ in range(steps):
                dev[state].append(eng.compute_resident(1)[1])
            launches[state] = eng.counts()["launches"]
            if state == "on":
                t0 = time.perf_counter()
                eng.atomic()
                fetch.append((time.perf_counter() - t0) * 1e3)
    prof = {}
    for state in ("off", "on"):
        eng.set_atomic(state == "on")
        eng.compute_resident(1)
        prof[state] = profile_final(eng, steps)
    c = eng.counts()
    eng.close()
    med = {s: float(np.median(v)) for s, v in dev.items()}
    spread = {s: [float(np.min(v)), float(np.max(v))] for s, v in dev.items()}
    return dict(family=family, atoms=len(atoms), edges=c["n_edges"], step_ms_median=med, step_ms_minmax=spread,
                overhead_pct=100.0 * (med["on"] / med["off"] - 1.0), fetch_ms_median=float(np.median(fetch)),
                launches=launches, final_kernels_ms=prof)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="chgnet:23,chgnet:50,tensornet:30",
                    help="family:cells list (C x C x C Si cells: 23 -> 97 336 atoms, 50 -> 1 M, 30 -> 216 000)")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    info = card()
    out = []
    for w in args.workloads.split(","):
        family, cells = w.split(":")
        r = run_workload(family, int(cells), args.rounds, args.steps, args.warmup)
        out.append(r)
        m, s = r["step_ms_median"], r["step_ms_minmax"]
        print(f"{family:9s} {r['atoms']:8d} atoms: off {m['off']:9.2f} ms [{s['off'][0]:.2f}, {s['off'][1]:.2f}]  "
              f"on {m['on']:9.2f} ms [{s['on'][0]:.2f}, {s['on'][1]:.2f}]  overhead {r['overhead_pct']:+.2f} %  "
              f"fetch {r['fetch_ms_median']:.1f} ms  launches {r['launches']}", flush=True)
        for state in ("off", "on"):
            print(f"    {state}: " + ", ".join(f"{k} {v:.3f} ms" for k, v in r["final_kernels_ms"][state].items()))
    print(f"card: {info}")
    print(json.dumps({"card": info, "workloads": out}))


if __name__ == "__main__":
    main()
