"""Diagnostic (not a test): wall time per structure-step of three ways to relax a batch of S 64-atom Si cells (random
strain +-3 %, perturbation 0.1 A), FIRE with the Frechet cell filter, for CHGNet, TensorNet and MACE "small":

  single  a loop of single-structure evaluations (b2m_set_structure + b2m_compute) with tests/relax_ref.py's FIRE
  host    relax_ref's FIRE over one b2m_compute_batch per step
  device  b2m_relax_batch (the loop on the device)

Random-weight models have no nearby minima at a usable fmax, so every arm runs a fixed number of steps with fmax = 0;
a last line per model shows compaction: the device loop with an fmax that half the structures reach, against fmax = 0.
Prints one JSON line per measurement, with the card's name and power limit read in the same run.
    python tests/relax_times.py [--S 64 1024] [--steps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distmlip_b200.structures import SimpleAtoms, si_diamond  # noqa: E402
from tests.relax_ref import relax  # noqa: E402
from tests.test_gpu_batch import Family  # noqa: E402


def cells(S, seed=0):
    rng = np.random.default_rng(seed)
    base = si_diamond(2, sigma=0.0)
    out = []
    for _ in range(S):
        strain = np.eye(3) + rng.uniform(-0.03, 0.03, (3, 3))
        x = base.get_positions() @ strain.T + rng.normal(0.0, 0.1, (len(base), 3))
        out.append(SimpleAtoms(base.get_chemical_symbols(), x, np.array(base.get_cell()) @ strain.T))
    return out


def inputs(fam, atoms):
    return ([len(a) for a in atoms], np.concatenate([a.get_positions() for a in atoms]),
            np.array([np.array(a.get_cell()) for a in atoms]), np.concatenate([fam.species(a) for a in atoms]),
            np.ones((len(atoms), 3), np.int32))


def host_batch_eval(fam, sym):
    def evaluate(ids, geos):
        fam.eng.set_structures([len(x) for x, _ in geos], np.concatenate([x for x, _ in geos]),
                               np.array([c for _, c in geos]), np.concatenate([fam.species(sym)] * len(geos)),
                               np.ones((len(geos), 3), np.int32))
        e, f, _ = fam.eng.compute_batch()
        _, w = fam.eng.atomic(virials=True)
        n = len(sym)
        return [(e[k], f[k * n:(k + 1) * n], w[k * n:(k + 1) * n].astype(np.float64).sum(0)) for k in range(len(geos))]
    return evaluate


def single_eval(fam, sym):
    fam.eng.set_atomic(True)

    def evaluate(ids, geos):
        out = []
        for x, c in geos:
            fam.eng.set_structure(x, c, fam.species(sym), np.ones(3, np.int32))
            e, f, _ = fam.eng.compute()
            _, w = fam.eng.atomic(virials=True)
            out.append((e, f, w.astype(np.float64).sum(0)))
        return out
    return evaluate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--S", type=int, nargs="+", default=[64, 1024])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--single-steps", type=int, default=2)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    for kind in ("chgnet", "tensornet", "mace_0e"):
        fam = Family(kind)
        for S in args.S:
            atoms = cells(S)
            sym = atoms[0]
            structs = [(a.get_positions(), np.array(a.get_cell())) for a in atoms]
            rows = {}
            fam.eng.relax_batch(*inputs(fam, atoms[:4]), fmax=0.0, steps=1)  # warm-up of every path
            t = time.perf_counter()
            relax(structs, single_eval(fam, sym), 0.0, args.single_steps, True)
            rows["single"] = (time.perf_counter() - t) / (S * (args.single_steps + 1))
            fam.eng.set_atomic(False)
            t = time.perf_counter()
            relax(structs, host_batch_eval(fam, sym), 0.0, args.steps, True)
            rows["host"] = (time.perf_counter() - t) / (S * (args.steps + 1))
            t = time.perf_counter()
            r = fam.eng.relax_batch(*inputs(fam, atoms), fmax=0.0, steps=args.steps)
            dev_all = time.perf_counter() - t
            rows["device"] = dev_all / (S * (args.steps + 1))
            print(json.dumps(dict(model=kind, S=S, natoms=len(sym), steps=args.steps, gpu=gpu,
                                  ms_per_structure_step={k: round(v * 1e3, 4) for k, v in rows.items()},
                                  device_ms_per_step=round(dev_all * 1e3 / (args.steps + 1), 3))), flush=True)
            # compaction: fmax at the median of the structures' final max atom-row forces, so that about half of them
            # stop early
            fm = np.sqrt((r["forces"].astype(np.float64) ** 2).sum(1)).reshape(S, -1).max(1)
            fmax = float(np.median(fm))
            t = time.perf_counter()
            rc = fam.eng.relax_batch(*inputs(fam, atoms), fmax=fmax, steps=args.steps)
            dt = time.perf_counter() - t
            evals = int((rc["steps"] + 1).sum())
            print(json.dumps(dict(model=kind, S=S, compaction=True, fmax=round(fmax, 4),
                                  converged=int(rc["converged"].sum()), evaluations=evals,
                                  ms_total=round(dt * 1e3, 2), ms_total_fmax0=round(dev_all * 1e3, 2), gpu=gpu)),
                  flush=True)


if __name__ == "__main__":
    main()
