"""MACE heat flux across processes, launched as
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tests/run_mace_heat_flux_multirank.py
Every rank drives one GPU and one slab of the unfolded cell; forces and per-atom energies are all-reduced with NCCL inside
libb200mlip before the contraction, so every rank must hold the same flux, and it must match the float64 oracle
(tests/mace_heat_flux_ref.py) for both hidden shapes with the ZBL pair term and the Agnesi transform."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distmlip_b200.implementations.mace import ScaleShiftMACE_Dist  # noqa: E402
from distmlip_b200.structures import si_diamond  # noqa: E402
from tests.mace_heat_flux_ref import heat_flux_ref  # noqa: E402
from tests.test_heat_flux_oracle_mace import mixed, model  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ok = True
    atoms = mixed(si_diamond(2, sigma=0.15, seed=11, nz=4 * world))
    v = np.random.default_rng(3).normal(scale=0.05, size=(len(atoms), 3))
    for shape in ("0e", "0e+1o"):
        make = lambda: model(shape, "zbl+agnesi", seed=4)  # noqa: E731
        dm = ScaleShiftMACE_Dist.from_existing(make())
        dm.enable_distributed_mode(list(range(world)))
        _e, _f, _s, _ae, _av, (j_pot, j_conv) = dm.evaluate_heat_flux(atoms, v)
        ok = ok and dm._engine.counts()["world"] == world
        if rank == 0:
            r = heat_flux_ref(make(), atoms, v)
            dp = np.abs(j_pot - r["j_pot"]).max() / r["scale"]
            dc = np.abs(j_conv - r["j_conv"]).max() / np.abs(v).sum()
            print(f"MACE {shape} world {world} natoms {len(atoms)}: |dJ_pot| / scale {dp:.2e}, |dJ_conv| / sum|v| "
                  f"{dc:.2e}", flush=True)
            ok = ok and dp < 1e-5 and dc < 2e-6
        t = torch.tensor(np.concatenate([j_pot, j_conv]), device="cuda")
        tmax, tmin = t.clone(), t.clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        ok = ok and float((tmax - tmin).abs().max()) == 0.0
        dm._engine.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("MACE HEAT FLUX MULTIRANK", "PASS" if flag.item() == 1 else "FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
