"""Diagnostic (not a test): what the balanced partition policy (DESIGN.md §4.1) buys, slab by slab, on one GPU.

    python tests/balance_times.py slabs [--quick] [--out FILE]   # per-slab resident step time, equal vs balanced
    python tests/balance_times.py graph [--cells 50]             # graph build time, equal vs balanced, alternating

`slabs`: every slab of a P-way split is timed alone through a b2m_set_partition view with the halo exchanges skipped
(B2M_DEBUG_NO_HALO=1, set here: right amount of per-partition work, wrong numbers), as tests/slab_timing.py does.  The
max over slabs is the compute floor of a P-GPU step (a step waits for its slowest partition); the step time of P GPUs
is not measured by this script.  Cells: two-phase (crystal + 3 % gas), particle in vacuum, uniform crystal (the
builders of tests/test_partition_balance.py).  One JSON line per (model, cell, P) and one with the card.
`graph`: the whole-structure graph build of one view (rank 0 of 4) at ~1 M atoms, the two policies alternating."""
import argparse
import json
import os
import subprocess
import sys

os.environ["B2M_DEBUG_NO_HALO"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from distmlip_b200 import _lib  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.test_partition_balance import particle, two_phase  # noqa: E402


def card():
    q = "--query-gpu=name,power.limit"
    return subprocess.run(["nvidia-smi", q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def chgnet():
    from distmlip_b200.random_init import RandomCHGNet

    sd = RandomCHGNet(seed=0).state_dict()
    eng = _lib.Engine(n_elem=sd["atom_embedding.weight"].shape[0], dim=64, max_n=9, max_f=4, n_blocks=4, cutoff=5.0,
                      three_body_cutoff=3.0, cutoff_exponent=5)
    eng.load_state_dict({k: v.float() for k, v in sd.items()})
    eng.finalize()
    return eng


def tensornet():
    from distmlip_b200.implementations.matgl import TensorNet_Dist
    from distmlip_b200.random_init import RandomTensorNet

    dm = TensorNet_Dist.from_existing(RandomTensorNet(seed=0))
    dm.enable_distributed_mode([0])
    dm._finalize(0.0, 1.0, None)
    return dm._engine


def mace_small():
    from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist
    from oracle.mace_ref import make_mace

    m = make_mace(seed=0, atomic_numbers=(14,), C=128, max_ell=3, correlation=3, num_interactions=2, r_max=6.0,
                  avg_num_neighbors=45.0)
    d = ScaleShiftMACE_Dist.from_existing(m)
    d.enable_distributed_mode([0])
    return d._engine


# (model, label, cells): ~100 k / ~1 M atoms for CHGNet, ~200 k for TensorNet, ~100 k for MACE "small"
def workloads(quick):
    c100 = {"two_phase": lambda: two_phase(16, 48, seed=1), "particle": lambda: particle(78.0, seed=1),
            "uniform": lambda: si_diamond(23, seed=1)}
    c1m = {"two_phase": lambda: two_phase(36, 96, seed=1), "particle": lambda: particle(168.0, seed=1),
           "uniform": lambda: si_diamond(50, seed=1)}
    c200 = {"two_phase": lambda: two_phase(20, 62, seed=1), "particle": lambda: particle(99.0, seed=1),
            "uniform": lambda: si_diamond(29, seed=1)}
    if quick:
        return [("chgnet", chgnet, {"two_phase": lambda: two_phase(6, 12, seed=1)})]
    return [("chgnet", chgnet, c100), ("tensornet", tensornet, c200), ("mace_small", mace_small, c100),
            ("chgnet", chgnet, c1m)]


def step_ms(eng, atoms, rank, world, policy, reps):
    eng.set_partition(rank, world)
    eng.set_partition_policy(policy)
    eng.set_structure(atoms.get_positions(), atoms.get_cell(), np.zeros(len(atoms), dtype=np.int32),
                      atoms.get_pbc().astype(np.int32))
    eng.compute_resident(2)
    ts = [eng.compute_resident(1)[1] for _ in range(reps)]
    return float(np.median(ts)), eng.counts()


def slabs(args):
    print(json.dumps({"card": card()}), flush=True)
    for model, make, cells in workloads(args.quick):
        eng = make()
        for cell, build in cells.items():
            atoms = build()
            one, _c = step_ms(eng, atoms, 0, 1, _lib.PARTITION_EQUAL, args.reps)
            for P in (2, 4, 8):
                rec = {"model": model, "cell": cell, "atoms": len(atoms), "P": P, "single_ms": round(one, 3)}
                for name, policy in (("equal", _lib.PARTITION_EQUAL), ("balanced", _lib.PARTITION_BALANCED)):
                    try:
                        res = [step_ms(eng, atoms, r, P, policy, args.reps) for r in range(P)]
                    except _lib.B2MError as e:
                        rec[name] = {"error": str(e)}
                        continue
                    ms = [t for t, _ in res]
                    rec[name] = {"max_ms": round(max(ms), 3), "mean_ms": round(float(np.mean(ms)), 3),
                                 "slab_ms": [round(t, 3) for t in ms],
                                 "edges": [c["n_edges"] for _, c in res], "angles": [c["n_angles"] for _, c in res]}
                print(json.dumps(rec), flush=True)
                if args.out:
                    with open(args.out, "a") as f:
                        f.write(json.dumps(rec) + "\n")
        eng.close()


def graph(args):
    """graph build of a 4-way view at rank 0, policies alternating, `reps` builds each"""
    print(json.dumps({"card": card()}), flush=True)
    eng = chgnet()
    atoms = si_diamond(args.cells, seed=1)
    out = {"atoms": len(atoms), "equal": [], "balanced": []}
    eng.set_partition(0, 4)
    for i in range(2 * args.reps + 2):
        name, policy = (("equal", _lib.PARTITION_EQUAL), ("balanced", _lib.PARTITION_BALANCED))[i % 2]
        eng.set_partition_policy(policy)
        eng.set_structure(atoms.get_positions(), atoms.get_cell(), np.zeros(len(atoms), dtype=np.int32),
                          atoms.get_pbc().astype(np.int32))
        if i >= 2:  # the first build of each allocates
            out[name].append(round(eng.timings()["graph_ms"], 3))
    for k in ("equal", "balanced"):
        out[k + "_median_ms"] = float(np.median(out[k]))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["slabs", "graph"])
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cells", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    slabs(a) if a.what == "slabs" else graph(a)
