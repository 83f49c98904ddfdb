"""CHGNet_Dist -- drop-in for DistMLIP.implementations.matgl.models.chgnet.CHGNet_Dist.

Same public surface (`from_existing`, `enable_distributed_mode`, `potential_forward_dist`), but the
forward/backward run in libb200mlip.so (hand-written sm_100a kernels) instead of PyTorch + DGL:

  reference                                                    here
  ---------------------------------------------------------    ------------------------------------------
  from_existing: shallow __dict__ copy   (chgnet.py:551-560)   same, plus a state_dict snapshot
  enable_distributed_mode: deep-copy 13 sub-modules per GPU    b2m_create + b2m_load_weights (one process
    from one Python thread               (chgnet.py:455-549)     per GPU; weights replicated, never sharded)
  potential_forward_dist + dist_forward  (chgnet.py:21-453)    b2m_compute on the resident graph

Two ways to use several GPUs, both behind the reference's call `enable_distributed_mode([0, 1, ...])`:
  * from ONE process (the reference's own usage, examples/chgnet_example.ipynb cell 1): a single-process group --
    one partition, host thread and stream per entry of `gpus`, halo rows exchanged as peer-memory stores;
  * under `torchrun` (torch.distributed initialised, world == len(gpus)): one process per GPU, rank r drives
    gpus[r], NCCL point-to-point halo exchange.
"cpu" entries are rejected: there is no CPU path in this engine.
"""
from __future__ import annotations

from distmlip_b200 import _lib

from ._base import EngineBackedModel


class CHGNet_Dist(EngineBackedModel):
    """Main CHGNet model (H100 engine behind the reference's wrapper API)."""

    __version__ = 1
    _has_site = True

    def heat_flux_reach(self):
        """max(n_blocks * r_cut, r_cut + (n_blocks - 1) * r_bond): a message moves r_cut per atom conv or r_bond per
        bond conv, and a bond feature reaches the atom graph only at its own bond's endpoint (DESIGN.md §10)"""
        nb, rc, rb = int(self._attr("n_blocks")), float(self._attr("cutoff")), float(self._attr("three_body_cutoff"))
        return max(nb * rc, rc + (nb - 1) * rb)

    def enable_distributed_mode(self, gpus, balance=False):
        """chgnet.py:455-549. `gpus`: CUDA ordinals, one per partition.  `balance`: place the slab walls so that every
        partition holds about the same number of edges and angles (DESIGN.md §4.1) instead of equally spaced."""
        gpus, rank, world, group = self._process_layout(gpus)
        sd = self._state_dict
        dim = int(sd["atom_embedding.weight"].shape[1])
        max_n = int(sd["bond_expansion.frequencies"].shape[0])
        max_f = int(sd["angle_expansion.frequencies"].shape[0]) - 1
        if not self._attr("use_bond_graph", True):
            raise NotImplementedError("use_bond_graph=False is not supported by the engine yet")
        if self._attr("state_embedding") is not None:
            raise NotImplementedError("State features not implemented for distributed computation.")
        if self._attr("readout_field", "atom_feat") not in ("atom_feat", "node_feat"):
            raise NotImplementedError("only atom_feat readout is supported (chgnet.py:442-449)")
        # the kernels hard-code SiLU hidden activations with a sigmoid gate and a sum readout (chgnet.py:436-438 honours
        # self.readout_operation; matgl's default activation_type is "swish")
        act = self._attr("activation_type", "swish")
        if isinstance(act, str) and act.lower() not in ("swish", "silu"):
            raise NotImplementedError(f"activation_type={act!r}: the engine implements swish/SiLU only")
        if str(self._attr("readout_operation", "sum")).lower() != "sum":
            raise NotImplementedError("readout_operation must be 'sum' (the engine sums atomic energies)")
        eng = _lib.Engine(
            n_elem=int(sd["atom_embedding.weight"].shape[0]), dim=dim, max_n=max_n, max_f=max_f,
            n_blocks=int(self._attr("n_blocks")), cutoff=float(self._attr("cutoff")),
            three_body_cutoff=float(self._attr("three_body_cutoff")),
            cutoff_exponent=int(self._attr("cutoff_exponent")),
            device=[int(g) for g in gpus] if group else int(gpus[rank]))
        self._attach_engine(eng, gpus, rank, world, group, balance)
