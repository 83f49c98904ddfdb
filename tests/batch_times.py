"""Diagnostic (not a test): cost of evaluating many small structures one call each against one batched call
(b2m_set_structures + b2m_compute_batch, DESIGN.md §12).  For CHGNet, TensorNet and MACE "small" (random weights of the
MACE-MP-0 small shape) on S perturbed 64-atom Si cells, each round times a loop of single calls (Potential_Dist.forward
/ ScaleShiftMACE_Dist.evaluate: graph build, evaluation, fetch) and one batched call over the same structures
(forward_batch / evaluate_batch), alternating the two in one process.  Reports medians over the rounds of host wall time
per structure, set_structures included, and the device time of the last call from b2m_last_timings (graph build,
forward + backward).  The card's name and power limit are read in the same run.  Prints a table and a last JSON line.

    python tests/batch_times.py [--sizes 1 64 1024] [--rounds 3] [--families chgnet,tensornet,mace_small]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.atomic_times import card  # noqa: E402


def model_of(family):
    """(single(atoms), batch(atoms_list), engine) of a one-GPU model with random weights"""
    if family == "mace_small":
        from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist
        from oracle.mace_ref import make_mace

        m = make_mace(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
                      avg_num_neighbors=45.0)
        d = ScaleShiftMACE_Dist.from_existing(m)
        d.enable_distributed_mode([0])
        return d.evaluate, d.evaluate_batch, d._engine
    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist, TensorNet_Dist
    from distmlip_b200.random_init import RandomCHGNet, RandomTensorNet

    dm = (CHGNet_Dist.from_existing(RandomCHGNet(seed=0)) if family == "chgnet"
          else TensorNet_Dist.from_existing(RandomTensorNet(seed=0)))
    dm.enable_distributed_mode([0])
    pot = Potential_Dist(model=dm)
    return pot.forward, pot.forward_batch, dm._engine


def device_ms(eng):
    t = eng.timings()
    return t["graph_ms"], t["fwd_ms"] + t["bwd_ms"]


def run(family, sizes, rounds):
    single, batch, eng = model_of(family)
    structures = [si_diamond(2, sigma=0.1, seed=1000 + k) for k in range(max(sizes))]
    single(structures[0])
    batch(structures[:2])  # warm-up: module loads, allocations
    out = []
    for S in sizes:
        atoms = structures[:S]
        batch(atoms)
        loop_ms, batch_ms = [], []
        for _r in range(rounds):
            t0 = time.perf_counter()
            for a in atoms:
                single(a)
            loop_ms.append((time.perf_counter() - t0) * 1e3 / S)
            loop_dev = device_ms(eng)
            t0 = time.perf_counter()
            batch(atoms)
            batch_ms.append((time.perf_counter() - t0) * 1e3 / S)
            batch_dev = device_ms(eng)
        r = dict(family=family, S=S, atoms=64 * S, loop_ms_per_structure=float(np.median(loop_ms)),
                 batch_ms_per_structure=float(np.median(batch_ms)),
                 loop_ms_minmax=[float(min(loop_ms)), float(max(loop_ms))],
                 batch_ms_minmax=[float(min(batch_ms)), float(max(batch_ms))],
                 single_call_device_ms={"graph": loop_dev[0], "fwd_bwd": loop_dev[1]},
                 batch_call_device_ms={"graph": batch_dev[0], "fwd_bwd": batch_dev[1]},
                 batch_launches=eng.counts()["launches"])
        r["speedup"] = r["loop_ms_per_structure"] / r["batch_ms_per_structure"]
        print(f"{family:10s} S={S:5d}: loop {r['loop_ms_per_structure']:8.3f} ms/structure "
              f"[{r['loop_ms_minmax'][0]:.3f}, {r['loop_ms_minmax'][1]:.3f}]  batch "
              f"{r['batch_ms_per_structure']:8.3f} ms/structure [{r['batch_ms_minmax'][0]:.3f}, "
              f"{r['batch_ms_minmax'][1]:.3f}]  x{r['speedup']:.1f}  device: single call graph {loop_dev[0]:.3f} + "
              f"{loop_dev[1]:.3f} ms, batch graph {batch_dev[0]:.3f} + {batch_dev[1]:.3f} ms", flush=True)
        out.append(r)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 64, 1024])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--families", default="chgnet,tensornet,mace_small")
    args = ap.parse_args()
    info = card()
    res = []
    for fam in args.families.split(","):
        res += run(fam, args.sizes, args.rounds)
    print(f"card: {info}")
    print(json.dumps({"card": info, "results": res}))


if __name__ == "__main__":
    main()
