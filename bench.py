#!/usr/bin/env python
"""bench.py -- atoms/s for one CHGNet energy+forces(+stress) evaluation on perturbed diamond Si.

  python bench.py --gpus N --steps K --warmup W            # our arm (libb200mlip, sm_90a)
  python bench.py --impl reference --steps K --warmup W    # reference arm: CPU restatement of the
                                                           # reference's path on the host cores

Contract (see the task statement): one JSON line on stdout from rank 0.
  value   = atoms / device time of forward+backward with the graph already resident in HBM
            (CUDA events on the engine's compute stream, max over ranks)
  e2e     = same metric through the public API (Potential_Dist.__call__) with HOST buffers:
            pinned host positions -> GPU graph build -> forward -> backward -> forces back to host
  roofline= edge-gather (atom conv forward) kernel, algorithmic bytes / event time / measured HBM peak
Workload (default, every N): the metric's own cell -- 50 x 50 x 50 conventional Si cells = 1 000 000 atoms, sliced
into N slabs ("scaling": "strong"; one 80 GB H100 holds it).  `--cells 23` runs BASELINE config[1] (97 336 atoms) the same
way; `--weak-cells n` grows an n x n x (n*N) cell with N instead ("scaling": "weak").  Activations per pass are GBs,
far larger than the 50 MB L2, so no explicit flush is needed between timed steps.
Every line carries a `parity` object computed in the run: net-force and virial-symmetry residuals, energy per atom,
a checksum of the forces of 4096 seeded atoms and -- at N > 1 -- the difference of E and of ALL forces against a
single-partition evaluation of the same cell done on rank 0's GPU outside the timed region.
`--dump-outputs DIR` writes, after the timed steps, what the last timed step computed (energy, forces, stress) as
DIR/<name>.npy; the inputs (structure, seeded weights) are the same in every run with the same arguments.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")  # keep stdout to the one JSON line (NCCL banner -> stderr)

METRIC = "atoms/sec (energy+forces) CHGNet a-Si r_cut=5A"
SURVEY_BYTES_PER_EDGE = 314.0  # SURVEY.md 8(d), rbf-recompute variant, D=64 fp32


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "NVIDIA H100 SXM data sheet (HBM3), not measured"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.rows = []
        self.proc = None

    def start(self, wait_first=5.0):
        """Launch the poller and wait for its first row: NVML start-up (up to a second on a fresh box) must not eat
        the timed region, which is only a few hundred milliseconds long."""
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50", "-i",
                 str(self.idx)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
            t0 = time.perf_counter()
            while not self.rows and time.perf_counter() - t0 < wait_first:
                time.sleep(0.01)
        except Exception:  # noqa: BLE001
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([time.perf_counter()] + [x.strip() for x in line.split(",")])

    def stop(self, windows):
        """windows: [(label, t_begin, t_end)] in perf_counter time; rows of the first window are used, the later ones
        (also under load) only if the first caught fewer than two samples."""
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "samples": 0}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:  # noqa: BLE001
            self.proc.kill()
        used, rows = [], []
        for label, tb, te in windows:
            rows += [r[1:] for r in self.rows if tb <= r[0] <= te]
            used.append(label)
            if len(rows) >= 2:
                break
        sm, smax, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            try:
                sm.append(float(r[1]))
                smax.append(float(r[2]))
                for k, nm in enumerate(names):
                    if r[5 + k].lower().startswith("active"):
                        reasons.add(nm)
            except Exception:  # noqa: BLE001
                pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "reasons": sorted(reasons), "samples": len(sm), "window": "+".join(used)}


def cpu_reference_step(n_cells, threads):
    """One bounded sample of the reference path on the host: the reference's own C graph builder
    (oracle/_ref, P=2, rebuilt every call as pes.py:69-85 does) + the PyTorch restatement of the model
    (forward + autograd backward).  Returns (atoms, seconds, detail)."""
    import torch

    from distmlip_b200.structures import si_diamond
    from oracle import graph_ref as G
    from oracle.chgnet_ref import CHGNetRef, build_line_graph

    torch.set_num_threads(threads)
    atoms = si_diamond(n_cells)
    cart, lat, pbc = atoms.get_positions(), atoms.get_cell(), atoms.get_pbc().astype(np.int64)
    t0 = time.perf_counter()
    kind = "port"
    t_graph = None
    builder = "numpy restatement of the reference's graph builder (oracle/graph_ref.py; oracle/_ref not built)"
    if G.load_ref_extension() is not None and n_cells >= 6:
        builder = "reference C graph builder (oracle/_ref, P=2)"
        frac = atoms.get_scaled_positions(wrap=True)
        ref = G.ref_get_subgraphs(cart, frac, lat, pbc, 2, 5.0, 3.0, True, num_threads=threads)
        t_graph = time.perf_counter() - t0
        i1, i2, off = ref[5], ref[6], np.rint(ref[7]).astype(np.int64)
        bond = np.zeros(len(i1), bool)
        bond[ref[11]] = True
    else:
        i1, i2, off, _d2, bond = G.neighbor_list(cart, lat, pbc, 5.0, 3.0)
        t_graph = time.perf_counter() - t0
    bond_edges, la, lb, ce = build_line_graph(i1, i2, bond)  # not timed: python loop, the reference does this in C
    model = cpu_reference_step.model = getattr(cpu_reference_step, "model", None) or CHGNetRef()
    t = lambda a: torch.as_tensor(a, dtype=torch.int64)
    lattice = torch.tensor(lat, dtype=torch.float32)
    t1 = time.perf_counter()
    strain = torch.zeros(3, 3, requires_grad=True)
    L = lattice @ (torch.eye(3) + strain)
    pos = torch.tensor(atoms.get_scaled_positions(False), dtype=torch.float32) @ L
    pos.retain_grad()
    vec = pos[t(i2)] + torch.tensor(off, dtype=torch.float32) @ L - pos[t(i1)]
    types = torch.full((len(atoms),), model.element_types.index("Si"), dtype=torch.int64)
    e, _ = model.forward_graph(pos, vec, t(i1), t(i2), t(bond_edges), t(la), t(lb), t(ce), types)
    e.backward()
    t_model = time.perf_counter() - t1
    return len(atoms), t_graph + t_model, {"graph_s": t_graph, "model_s": t_model, "kind": kind, "graph_builder": builder}


def best_thread_count(n_cells=8):
    """PyTorch CPU ops on these tensors stop scaling past a few dozen threads; pick the fastest of a few thread counts
    (up to every host core) on the SAME sample size the baseline is then timed on, so the CPU arm is not handicapped
    on many-core hosts.  Returns (threads, {threads: seconds})."""
    cores = os.cpu_count() or 1
    # (beyond 64 threads these small tensors get dramatically slower, so the probe stops there instead of spending a
    #  minute to confirm it)
    cands = sorted({c for c in (8, 16, 32, 64) if c <= cores}) or [cores]
    best, best_t, seen = cands[0], 1e30, {}
    cpu_reference_step(n_cells, cands[0])  # first call pays imports / allocator warm-up
    for c in cands:
        _a, sec, _d = cpu_reference_step(n_cells, c)
        seen[c] = round(sec, 3)
        if sec < best_t:
            best, best_t = c, sec
    return best, seen


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    n_cells = 10  # 8000 atoms: a bounded sample of the same structure family
    cores, probe = best_thread_count(n_cells)
    for _ in range(max(1, min(args.warmup, 1))):
        cpu_reference_step(n_cells, cores)
    ts, atoms = [], 0
    for _ in range(args.steps):
        atoms, sec, det = cpu_reference_step(n_cells, cores)
        ts.append(sec)
    sec = float(np.mean(ts))
    val = atoms / sec
    sample = (f"{atoms}-atom perturbed diamond Si ({n_cells}x{n_cells}x{n_cells} cells), {det['graph_builder']} "
              f"({det['graph_s']:.2f}s) + PyTorch-CPU restatement fwd+autograd bwd ({det['model_s']:.2f}s); {cores} threads = "
              f"fastest of {probe} s/step on this sample (host has {os.cpu_count()} cores)")
    line = {
        "impl": "reference", "metric": METRIC, "value": val, "unit": "atoms/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True,
        "scaling": "weak" if args.weak_cells > 0 else "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "CHGNet energy+forces+stress, perturbed diamond Si, r_cut=5A r_bond=3A",
                   "note": "bounded CPU sample (8000 atoms) of the same workload family; atoms/s of this path is size "
                           "independent above a few thousand atoms"},
        "cpu_baseline": {"value": val, "unit": "atoms/s", "cores": cores, "kind": "port", "graph_builder": det["graph_builder"],
                         "sample": sample},
        "e2e": {"value": val, "unit": "atoms/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def parity_block(atoms, out, pot_factory, rank, world, local, release=None):
    """Correctness evidence computed in the run (outside the timed region).  Always: net force, virial symmetry,
    energy per atom, checksum of the forces of 4096 seeded atoms.  At N > 1 rank 0 also evaluates the same cell on a
    single partition (its own GPU, a second engine) and reports the difference of E and of every force component."""
    import torch

    E, F, S = float(out[0].item()), out[1].numpy(), out[2].numpy()
    n = len(atoms)
    ids = np.random.default_rng(1234).choice(n, size=min(4096, n), replace=False)
    blk = {
        "energy_per_atom": E / n,
        "net_force_max": float(np.abs(F.astype(np.float64).sum(0)).max()),
        "f_abs_max": float(np.abs(F).max()),
        "virial_asym_max": float(np.abs(S - S.T).max()),
        "f_probe_l1": float(np.abs(F[ids].astype(np.float64)).sum()),
        "finite": bool(np.isfinite(F).all() and np.isfinite(E)),
        "tolerance": "north_star: 1e-4 eV/atom, 1e-3 eV/A",
    }
    if world > 1 and rank == 0:
        try:
            if release is not None:
                release()  # this rank's own partition is not needed any more: give its memory to the check
            free, _tot = torch.cuda.mem_get_info()
            pot1 = pot_factory()
            o1 = pot1(atoms)
            blk["vs_single_partition"] = {
                "dE_per_atom": abs(E - float(o1[0].item())) / n,
                "dF_max": float(np.abs(F - o1[1].numpy()).max()),
                "dS_max": float(np.abs(S - o1[2].numpy()).max()),
                "free_gb_before": round(free / 1e9, 1),
            }
            pot1.model._engine.close()
        except Exception as ex:  # noqa: BLE001  (out of memory next to this rank's own partition: say so)
            blk["vs_single_partition"] = {"skipped": str(ex)[:200]}
    return blk


def dump_outputs(out_dir, eng):
    """energy, forces and stress of the engine's last evaluation, as a caller of the timed path receives them"""
    e, f, s = eng.results()
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "energy.npy"), np.array([e], dtype=np.float64))
    np.save(os.path.join(out_dir, "forces.npy"), np.ascontiguousarray(f, dtype=np.float32))
    np.save(os.path.join(out_dir, "stress.npy"), np.ascontiguousarray(s, dtype=np.float32))


def run_ours(args):
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run --nproc-per-node N for --gpus N")
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    from distmlip_b200.implementations.matgl import CHGNet_Dist, Potential_Dist, TensorNet_Dist
    from distmlip_b200.structures import si_diamond
    from distmlip_b200.random_init import RandomCHGNet, RandomTensorNet  # seeded random-init weights of the architectures

    tn = args.model == "tensornet"  # SURVEY 8(f).2, not the metric's model: a reduced line (no roofline / cpu_baseline)

    strong = args.weak_cells <= 0
    if args.rough_atoms > 0:  # degree-imbalanced stress structure (SURVEY 8d): random sequential addition, not the metric
        from distmlip_b200.structures import SimpleAtoms, rough_cell

        n = 0
        base = rough_cell(max(64, args.rough_atoms // (8 * world)), seed=0)  # python generator: build 1/8 and tile 2x2x(2 world)
        reps = (2, 2, 2 * world)
        lat, pos = base.get_cell(), base.get_positions()
        shifts = np.array([[i, j, k] for i in range(reps[0]) for j in range(reps[1]) for k in range(reps[2])], dtype=float) @ lat
        atoms = SimpleAtoms(base.get_chemical_symbols() * len(shifts), (pos[None] + shifts[:, None]).reshape(-1, 3),
                            lat * np.array(reps)[:, None])
    elif strong:  # default: fixed total cell (50 -> the metric's 1 000 000-atom cell), sliced across the ranks
        # TensorNet keeps ~5.9 KB per edge (DESIGN.md 8): the 1 M-atom cell does not fit an 80 GB H100, 30^3 cells do
        n = args.cells if args.cells is not None else (30 if tn else 50)
        atoms = si_diamond(n)
    else:       # fixed work per GPU, the cell grows along z with the number of ranks
        n = args.weak_cells
        atoms = si_diamond(n, nz=n * world)
    natoms = len(atoms)
    make = (lambda: TensorNet_Dist.from_existing(RandomTensorNet(seed=0))) if tn else \
           (lambda: CHGNet_Dist.from_existing(RandomCHGNet(seed=0)))
    model = make()
    model.enable_distributed_mode(list(range(world)) if world > 1 else [local])
    pot = Potential_Dist(model=model, calc_forces=True, calc_stresses=True)
    eng = model._engine

    def single_partition_potential():
        m1 = make()
        m1.enable_distributed_mode([local])  # one GPU, one partition (replica mode inside a multi-rank job)
        return Potential_Dist(model=m1, calc_forces=True, calc_stresses=True)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- resident-graph throughput (`value`) ----
    out = pot(atoms)  # builds graph + first compute
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    for _ in range(args.warmup):
        eng.compute_resident(1)
    barrier()
    t0 = time.perf_counter()
    dev_ms, gather_ms, launches = 0.0, [], 0
    for _ in range(args.steps):
        _e, ms = eng.compute_resident(1)
        dev_ms += ms
        gather_ms.append(eng.timings()["edge_gather_ms"])
        launches += eng.counts()["launches"]
    barrier()
    t1 = time.perf_counter()
    wall_ms = (t1 - t0) * 1e3
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, eng)
    tmax = torch.tensor([dev_ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    ms_per_step = tmax.item() / args.steps
    value = natoms / (ms_per_step * 1e-3)

    # ---- end to end through the public API, host buffers in, forces out ----
    # (Engine.set_structure stages positions/species through page-locked host buffers)
    for _ in range(max(1, min(args.warmup, 2))):
        pot(atoms)
    barrier()
    t2b = time.perf_counter()
    for _ in range(args.steps):
        out = pot(atoms)
        _ = float(out[0].item()) + float(out[1][0, 0])
    barrier()
    t2e = time.perf_counter()
    e2e_ms = (t2e - t2b) * 1e3 / args.steps
    clocks = sampler.stop([("timed", t0, t1), ("e2e", t2b, t2e)]) if rank == 0 else None
    t2 = torch.tensor([e2e_ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t2, op=dist.ReduceOp.MAX)
    e2e_ms = t2.item()
    e2e_val = natoms / (e2e_ms * 1e-3)
    c_final, tm = eng.counts(), eng.timings()
    parity = parity_block(atoms, out, single_partition_potential, rank, world, local, release=eng.release_workspace)
    barrier()

    if rank == 0 and tn:
        c = c_final
        print(json.dumps({
            "metric": "TensorNet energy+forces+stress throughput (not the headline metric)", "value": value, "unit": "atoms/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step,
            "higher_is_better": True, "scaling": "strong" if strong else "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": {"workload": f"TensorNet (matgl defaults: units 64, 2 blocks, 32 Gaussian rbf, O(3); random-init seed 0) "
                                   f"on {natoms}-atom perturbed diamond Si, r_cut=5A", "atoms": natoms,
                       "edges_per_gpu": c["n_edges"], "parallelism": f"slab{world}"},
            "phase_ms": {"graph_build": tm["graph_ms"], "forward": tm["fwd_ms"], "backward": tm["bwd_ms"]},
            "gpu_launches": launches, "clocks": clocks, "parity": parity,
            "e2e": {"value": e2e_val, "unit": "atoms/s", "ms_per_step": e2e_ms,
                    "h2d_bytes_per_step": natoms * (24 + 4) + 72 + 12, "d2h_bytes_per_step": natoms * 12 + 8 + 36}}), flush=True)
    elif rank == 0:
        c = c_final
        peak, peak_src = load_peaks()
        g_ms = float(np.mean(gather_ms))
        alg_bytes = SURVEY_BYTES_PER_EDGE * c["n_edges"]
        n_loc, n_own = c["n_own"] + c["n_halo"], c["n_own"]
        # own layout: indices+vec4 28 B per edge (the radial basis is recomputed in the kernel, nothing is saved for the
        # backward); A rows, C rows, agg, Q rows per node/bond
        own_bytes = 28.0 * c["n_edges"] + 512.0 * n_loc + 512.0 * n_own + 256.0 * n_own + 0.75 * 512.0 * c["n_bond_own"]
        achieved = alg_bytes / (g_ms * 1e-3) / 1e9
        line = {
            "metric": METRIC, "value": value, "unit": "atoms/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong" if strong else "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": (f"CHGNet (random-init, seed 0) energy+forces+stress on {natoms}-atom perturbed "
                                    f"diamond Si ({n}x{n}x{n if strong else n * world} cells, sigma 0.15 A), r_cut=5A r_bond=3A, "
                                    f"graph resident for `value`, rebuilt from host positions every step for `e2e`")
                       if args.rough_atoms <= 0 else
                       (f"NOT the metric's cell: CHGNet on a {natoms}-atom random-sequential-addition Si structure "
                        f"(min distance 2.2 A, 0.05 atoms/A^3; 10-40 edges and 0-12 bonds per atom), r_cut=5A r_bond=3A"),
                       "atoms": natoms, "atoms_per_gpu": natoms // world, "edges_per_gpu": c["n_edges"],
                       "angles_per_gpu": c["n_angles"], "parallelism": f"slab{world}",
                       "cache": "activations per pass >> 50 MB L2 (no explicit flush needed)"},
            "value_note": "device time of forward+backward on the resident graph; `e2e` (host positions in, graph rebuilt every "
                          "step, forces out) is the figure comparable with the reference arm, whose steps include its graph build",
            "wall_ms_per_step": wall_ms / args.steps,
            "phase_ms": {"graph_build": tm["graph_ms"], "forward": tm["fwd_ms"], "backward": tm["bwd_ms"]},
            "gpu_launches": launches,
            "clocks": clocks,
            "parity": parity,
            "e2e": {"value": e2e_val, "unit": "atoms/s", "ms_per_step": e2e_ms,
                    "h2d_bytes_per_step": natoms * (24 + 4) + 72 + 12, "d2h_bytes_per_step": natoms * 12 + 8 + 36 + natoms * 4},
            "roofline": {"bound": "hbm", "kernel": "k_atomconv_fwd (edge gather: bulk-copy-staged A[src] rows, FP32 FFMA)", "achieved": achieved,
                         "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                         "bytes_per_launch": alg_bytes, "bytes_convention": "SURVEY 8(d): 314 B/edge",
                         "kernel_ms": g_ms, "achieved_own_layout": own_bytes / (g_ms * 1e-3) / 1e9},
        }
        if world == 1 and not args.no_cpu_baseline:
            cores, probe = best_thread_count(8)
            a, sec, det = cpu_reference_step(8, cores)
            line["cpu_baseline"] = {
                "value": a / sec, "unit": "atoms/s", "cores": cores, "kind": "port", "graph_builder": det["graph_builder"],
                "sample": f"{a}-atom Si (8x8x8), {cores} threads = fastest of {probe} s/step on this sample (host has "
                          f"{os.cpu_count()} cores), {det['graph_builder']} {det['graph_s']:.2f}s + PyTorch-CPU "
                          f"restatement fwd+bwd {det['model_s']:.2f}s"}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--cells", type=int, default=None,
                    help="strong scaling (default): a fixed C x C x C cell for every N (50 -> the metric's 1 000 000 atoms; "
                         "23 -> 97 336 = BASELINE config[1]); default 50 for CHGNet, 30 (216 000 atoms) for TensorNet")
    ap.add_argument("--weak-cells", type=int, default=0,
                    help="weak scaling instead: n x n x (n*N) cells, i.e. fixed work per GPU (0 = off)")
    ap.add_argument("--rough-atoms", type=int, default=0,
                    help="time the degree-imbalanced random-sequential-addition structure with this many atoms instead")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--model", default="chgnet", choices=["chgnet", "tensornet"],
                    help="tensornet: the SURVEY 8(f).2 path (reduced JSON line; the metric and the default are CHGNet)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the energy, forces and stress of the last one as DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
