"""Heat flux across processes, launched as
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tests/run_heat_flux_multirank.py
Every rank drives one GPU and one slab of the unfolded cell; forces and per-atom energies are all-reduced with NCCL inside
libb200mlip before the contraction, so every rank must hold the same flux, and it must match the float64 oracle
(oracle/heat_flux_ref.py) for CHGNet and TensorNet."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist, TensorNet_Dist  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from oracle.heat_flux_ref import heat_flux_ref  # noqa: E402
from tests._util import make_model  # noqa: E402
from tests.test_oracle_tensornet import make_tn  # noqa: E402


class Moving:
    """Atoms with velocities (all silicon) for Potential_Dist"""

    def __init__(self, a, v):
        self.a, self.v = a, v

    def __getattr__(self, name):
        return getattr(self.a, name)

    def get_velocities(self):
        return self.v.copy()

    def get_masses(self):
        return np.full(len(self.v), 28.085)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ok = True
    atoms = si_diamond(2, sigma=0.15, seed=11, nz=4 * world)
    v = np.random.default_rng(3).normal(scale=0.05, size=(len(atoms), 3))
    for family in ("chgnet", "tensornet"):
        make = (lambda: make_model(seed=2)) if family == "chgnet" else (lambda: make_tn(seed=3, scale=1.5))
        dm = (CHGNet_Dist if family == "chgnet" else TensorNet_Dist).from_existing(make())
        dm.enable_distributed_mode(list(range(world)))
        pot = Potential_Dist(model=dm, data_mean=0.7, data_std=1.3, calc_heat_flux=True)
        pot(Moving(atoms, v))
        j_pot = pot.heat_flux["potential"]
        if rank == 0:
            r = heat_flux_ref(make(), atoms, v, data_mean=0.7, data_std=1.3)
            dp = np.abs(j_pot - r["j_pot"]).max() / r["scale"]
            print(f"{family} world {world} natoms {len(atoms)}: |dJ_pot| / scale {dp:.2e}", flush=True)
            ok = ok and dp < 1e-5
        t = torch.tensor(np.concatenate([j_pot, pot.heat_flux["convective"]]), device="cuda")
        tmax, tmin = t.clone(), t.clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        ok = ok and float((tmax - tmin).abs().max()) == 0.0
        dm._engine.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("HEAT FLUX MULTIRANK", "PASS" if flag.item() == 1 else "FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
