"""Per-atom energies and virials across processes, launched as
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tests/run_atomic_multirank.py
Every rank drives one GPU; the per-atom arrays are all-reduced with NCCL inside libb200mlip, so every rank must hold the
same arrays, and they must match the single-graph oracle (oracle/atomic_ref.py) for CHGNet and TensorNet."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist, TensorNet_Dist  # noqa: E402
from distmlip_b200.structures import SimpleAtoms, si_diamond  # noqa: E402
from oracle.atomic_ref import atomic_ref  # noqa: E402
from tests._util import make_model  # noqa: E402
from tests.test_oracle_tensornet import make_tn  # noqa: E402

GPA_PER_EVA3 = 160.21766208


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ok = True
    a0 = si_diamond(2, sigma=0.15, seed=11, nz=4 * world)
    atoms = SimpleAtoms(["O" if i % 3 == 0 else s for i, s in enumerate(a0.get_chemical_symbols())],
                        a0.get_positions(), a0.get_cell())
    for family in ("chgnet", "tensornet"):
        make = (lambda: make_model(seed=2)) if family == "chgnet" else (lambda: make_tn(seed=3, scale=1.5))
        refs = np.linspace(-0.5, 0.5, len(make().element_types))
        dm = (CHGNet_Dist if family == "chgnet" else TensorNet_Dist).from_existing(make())
        dm.enable_distributed_mode(list(range(world)))
        pot = Potential_Dist(model=dm, data_mean=0.7, data_std=1.3, element_refs=refs, calc_atomic=True)
        E, _F, S, _ = pot(atoms)
        eps = pot.atomic_energies.numpy()
        w = pot.atomic_stresses.numpy().astype(np.float64) * atoms.get_volume() / GPA_PER_EVA3
        if rank == 0:
            r = atomic_ref(make(), atoms, data_mean=0.7, data_std=1.3, element_refs=refs, dtype=torch.float64)
            de = np.abs(eps - r["energies"].numpy()).max()
            dw = np.abs(w - r["virials"].numpy()).max()
            se = abs(eps.sum() - float(E)) / abs(float(E))
            ss = np.abs(pot.atomic_stresses.double().sum(0).numpy() - S.double().numpy()).max()
            print(f"{family} world {world} natoms {len(atoms)}: max|d eps| {de:.2e} max|d w| {dw:.2e} "
                  f"sum eps rel {se:.2e} sum sigma {ss:.2e} GPa", flush=True)
            ok = ok and de < 1e-4 and dw < 5e-3 and se < 1e-6 and ss < 1e-5 * float(S.abs().max()) + 1e-6
        # every rank holds the same (all-reduced) arrays
        t = torch.tensor(np.concatenate([eps, pot.atomic_stresses.numpy().ravel()]), device="cuda")
        tmax, tmin = t.clone(), t.clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        ok = ok and float((tmax - tmin).abs().max()) == 0.0
        dm._engine.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("ATOMIC MULTIRANK", "PASS" if flag.item() == 1 else "FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
