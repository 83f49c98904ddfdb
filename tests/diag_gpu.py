"""Stage-by-stage GPU diagnostic (not a pytest file): prints max errors of every tap vs the oracle.
Usage on a GPU machine:  python tests/diag_gpu.py [ncells]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests._util import *  # noqa

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2
torch.set_num_threads(os.cpu_count())
model = make_model()
atoms = si_diamond(n)
og = oracle_graph(atoms)
print(f"atoms {len(atoms)} edges {len(og['i1'])} bonds {len(og['bond_edges'])} angles {len(og['la'])}", flush=True)
eng = engine_from_model(model)
species = np.array([model.element_types.index(s) for s in atoms.get_chemical_symbols()], dtype=np.int32)
eng.set_structure(atoms.get_positions(), atoms.get_cell(), species, atoms.get_pbc().astype(np.int32))
c = eng.counts()
print("counts", c, flush=True)
ok = c["n_edges"] == len(og["i1"]) and c["n_bond_own"] == len(og["bond_edges"]) and c["n_angles"] == len(og["la"])
print("graph counts match:", ok, flush=True)
ep, bp, ap = maps_to_oracle(eng, og)
print("graph maps ok (all engine rows found in oracle); unique:",
      len(set(ep)) == len(ep), len(set(bp)) == len(bp), len(set(ap)) == len(ap), flush=True)
gid = eng.partition_info(0)
ev = eng.debug_tensor("e_vec")
print("e_vec max err", np.abs(ev[:, :3] - og["vec"][ep]).max(), "d err", np.abs(ev[:, 3] - np.sqrt(og["d2"][ep])).max())

E, F, S = eng.compute(True, True)
print("timings", eng.timings(), "launches", eng.counts()["launches"], flush=True)
ref = manual_run(model, atoms, og)
taps = ref["taps"]


def cmp(name, mine, theirs):
    theirs = theirs.numpy() if hasattr(theirs, "numpy") else theirs
    err = np.abs(mine - theirs).max()
    print(f"  {name:8s} max|err| {err:.3e}   max|ref| {np.abs(theirs).max():.3e}  nan={np.isnan(mine).any()}", flush=True)


for l in range(model.n_blocks + 1):
    if f"x{l}" in taps:
        cmp(f"x{l}", eng.debug_tensor(f"x{l}"), taps[f"x{l}"][gid])
for l in range(model.n_blocks):
    if f"h{l}" in taps:
        cmp(f"h{l}", eng.debug_tensor(f"h{l}"), taps[f"h{l}"][bp])
for l in range(model.n_blocks - 1):
    if f"ang{l}" in taps:
        cmp(f"ang{l}", eng.debug_tensor(f"ang{l}"), taps[f"ang{l}"][ap])
cmp("e_atom", eng.debug_tensor("e_atom")[:, 0], taps["e_atom"][gid, 0])
gd_e = eng.debug_tensor("gd")[:, 0].copy()
gdb = eng.debug_tensor("gdb")[:, 0]
bkeys = {k: i for i, k in enumerate(key5(eng.partition_info(4)))}
for i, k in enumerate(key5(eng.partition_info(3))):
    if k in bkeys:
        gd_e[i] += gdb[bkeys[k]]
cmp("gd", gd_e, taps["gd"][ep])  # oracle gd includes the bond-node part
cmp("gbvec", eng.debug_tensor("gbvec"), taps["gbvec"][bp])
cmp("gh0", eng.debug_tensor("gh"), taps["gh0"][bp])
cmp("gang0", eng.debug_tensor("gang"), taps["gang0"][ap])
Fm, Sm = M.forces_from_gvec(ref["gvec"], og["vec"], og["i1"], og["i2"], len(atoms), atoms.get_volume())
print(f"E engine {E:.8f}  oracle {ref['energy'].item():.8f}  dE/atom {abs(E - ref['energy'].item()) / len(atoms):.3e}")
print(f"F max err {np.abs(F - Fm.numpy()).max():.3e}  max|F| {np.abs(Fm.numpy()).max():.3e}")
print(f"S max err {np.abs(S - Sm.numpy()).max():.3e}  max|S| {np.abs(Sm.numpy()).max():.3e}")
Ea, Fa, Sa, _ = potential_ref(model, atoms, dtype=torch.float32)
print(f"vs autograd fp32 oracle: dE/atom {abs(E - Ea.item()) / len(atoms):.3e} dF {np.abs(F - Fa.numpy()).max():.3e} dS {np.abs(S - Sa.numpy()).max():.3e}")
