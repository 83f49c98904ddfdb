"""MACE with hidden features 0e+1o, one process per GPU (NCCL halo exchange of the 4 C-wide node features and
all-reduce of the results), launched as
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tests/run_mace_eq_multirank.py
Every rank drives one GPU; every rank must hold the same energy, forces, stress and per-atom values, and they must match
the f64 oracle (tests/mace_eq_ref.py)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.structures import SimpleAtoms, si_diamond  # noqa: E402
from tests.mace_eq_ref import atomic_virials_ref, make_mace_eq, potential_ref  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    a0 = si_diamond(2, sigma=0.15, seed=11, nz=6 * world)
    atoms = SimpleAtoms(["O" if i % 3 == 0 else ("C" if i % 5 == 0 else s) for i, s in enumerate(a0.get_chemical_symbols())],
                        a0.get_positions(), a0.get_cell())
    make = lambda: make_mace_eq(seed=4, C=32, r_max=5.0, scale=8.0, num_interactions=3)  # noqa: E731
    dm = ScaleShiftMACE_Dist.from_existing(make())
    dm.enable_distributed_mode(list(range(world)))
    e, f, s, ae, av = dm.evaluate(atoms, atomic=True)
    ok = dm._engine.counts()["world"] == world
    if rank == 0:
        E, F, S, eps = potential_ref(make(), atoms)
        w = atomic_virials_ref(make(), atoms)
        de = abs(e - E.item()) / len(atoms)
        df = np.abs(f - F.numpy()).max()
        ds = np.abs(s - S.numpy()).max()
        dw = np.abs(av - w.numpy()).max()
        da = np.abs(ae - eps.numpy()).max()
        print(f"MACE 0e+1o world {world} natoms {len(atoms)}: dE/atom {de:.2e} dF {df:.2e} dS {ds:.2e} d eps {da:.2e} "
              f"d w {dw:.2e}", flush=True)
        ok = ok and de < 1e-4 and df < 1e-3 and ds < 1e-3 and da < 1e-4 and dw < 1e-3
    t = torch.tensor(np.concatenate([[e], f.ravel(), s.ravel(), ae, av.ravel()]), device="cuda")
    tmax, tmin = t.clone(), t.clone()
    dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
    ok = ok and float((tmax - tmin).abs().max()) == 0.0
    dm._engine.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("MACE EQ MULTIRANK", "PASS" if flag.item() == 1 else "FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
