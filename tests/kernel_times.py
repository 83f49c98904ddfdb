"""Diagnostic (not a test): per-kernel device time of one CHGNet energy+forces+stress step on the resident graph of the
perturbed diamond Si cell that bench.py times (one GPU, one partition), from torch.profiler with CUDA activities.
Prints one table row per kernel (launches / step, ms / step, share) and a last JSON line with the same numbers and the
card's name, power limit and SM clock limit.

    python tests/kernel_times.py [--cells 23] [--steps 5] [--warmup 3] [--trace DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200 import _lib  # noqa: E402
from distmlip_b200.random_init import RandomCHGNet  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:100]}


def short_name(name):
    """kernel symbol -> the name used in DESIGN's tables (template arguments kept, namespaces and parameters dropped)"""
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*\)$", "", name)
    return name.replace("b2m::", "")


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=23, help="C x C x C conventional Si cells (23 -> 97 336 atoms, 50 -> 1 M)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", default=None, help="also write a Chrome trace into this directory")
    args = ap.parse_args()

    sd = RandomCHGNet(seed=0).state_dict()
    eng = _lib.Engine(n_elem=sd["atom_embedding.weight"].shape[0], dim=64, max_n=9, max_f=4, n_blocks=4, cutoff=5.0,
                      three_body_cutoff=3.0, cutoff_exponent=5)
    eng.load_state_dict({k: v.float() for k, v in sd.items()})
    eng.finalize()
    atoms = si_diamond(args.cells)
    eng.set_structure(atoms.get_positions(), atoms.get_cell(), np.zeros(len(atoms), dtype=np.int32),
                      atoms.get_pbc().astype(np.int32))
    for _ in range(args.warmup):
        eng.compute_resident(1)
    torch.cuda.synchronize()
    step_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step_ms.append(eng.compute_resident(1)[1])
        torch.cuda.synchronize()
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace, f"kernel_times_c{args.cells}.pt.trace.json"))

    tot, cnt = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = short_name(ev.name)
            tot[k] += ev.device_time_total / 1e3  # us -> ms
            cnt[k] += 1
    allk = sum(tot.values())
    c = eng.counts()
    info = card()
    print(f"{len(atoms)} atoms, {c['n_edges']} edges, {c['n_angles']} angles; {info}")
    print(f"step (CUDA events, profiler on): {np.mean(step_ms):.2f} ms; kernels sum {allk / args.steps:.2f} ms/step")
    rows = sorted(tot, key=lambda k: -tot[k])
    for k in rows:
        print(f"  {k:60s} {cnt[k] / args.steps:6.1f} launches  {tot[k] / args.steps:9.3f} ms/step  {100 * tot[k] / allk:5.1f} %")
    print(json.dumps({"atoms": len(atoms), "edges": c["n_edges"], "steps": args.steps, "card": info,
                      "step_ms": float(np.mean(step_ms)),
                      "kernels": {k: {"launches_per_step": cnt[k] / args.steps, "ms_per_step": tot[k] / args.steps}
                                  for k in rows}}))
    eng.close()


if __name__ == "__main__":
    main()
