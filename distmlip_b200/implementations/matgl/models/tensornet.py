"""TensorNet_Dist -- drop-in for DistMLIP.implementations.matgl.models.tensornet.TensorNet_Dist.

Same public surface (`from_existing`, `enable_distributed_mode`, `potential_forward_dist`); the forward and the reverse
pass run in libb200mlip.so (csrc/kernels_tn.cu) instead of PyTorch + DGL:

  reference                                                          here
  ---------------------------------------------------------------    ------------------------------------------
  from_existing: shallow __dict__ copy        (tensornet.py:206-217)  same, plus a state_dict snapshot
  enable_distributed_mode: deep copies of bond_expansion,             b2m_create_tensornet + b2m_load_weights
    tensor_embedding, layers per GPU; linear, final_layer,              (weights replicated per partition)
    out_norm on gpus[0]                       (tensornet.py:163-204)
  potential_forward_dist + dist_forward       (tensornet.py:10-147)   b2m_compute on the resident graph

Supported configuration (anything else raises): units = 64, Gaussian bond expansion with at most 64 centres, swish,
"O(3)" or "SO(3)", is_intensive = False (the reference raises for True as well, tensornet.py:139-142), no state features.
"""
from __future__ import annotations

from distmlip_b200 import _lib

from ._base import EngineBackedModel


class TensorNet_Dist(EngineBackedModel):
    """TensorNet model (H100 engine behind the reference's wrapper API)."""

    __version__ = 1

    def heat_flux_reach(self):
        """(n_blocks + 1) * r_cut: the embedding aggregates one hop, every interaction layer one more"""
        nblocks = len({int(k.split(".")[1]) for k in self._state_dict if k.startswith("layers.")})
        return (nblocks + 1) * float(self._attr("cutoff"))

    def enable_distributed_mode(self, gpus, balance=False):
        """tensornet.py:163-204. `gpus`: CUDA ordinals, one per partition.  `balance`: place the slab walls so that
        every partition holds about the same number of edges (DESIGN.md §4.1) instead of equally spaced."""
        gpus, rank, world, group = self._process_layout(gpus)
        sd = self._state_dict
        if self._attr("is_intensive", False):
            raise NotImplementedError("self.is_intensive = True is not yet supported by distributed inference")
        act = self._attr("activation_type", "swish")
        if isinstance(act, str) and act.lower() not in ("swish", "silu"):
            raise NotImplementedError(f"activation_type={act!r}: the engine implements swish/SiLU only")
        rbf_type = self._attr("rbf_type", None) or getattr(self._attr("bond_expansion"), "rbf_type", "Gaussian")
        if str(rbf_type) != "Gaussian" or "bond_expansion.rbf.centers" not in sd:
            raise NotImplementedError(f"rbf_type={rbf_type!r}: the engine implements the Gaussian bond expansion only")
        group_name = self._attr("equivariance_invariance_group")
        if group_name is None:  # matgl keeps the group on the interaction layers
            layers_mod = self._attr("layers")
            first = layers_mod[0] if layers_mod is not None and len(layers_mod) else None
            group_name = getattr(first, "equivariance_invariance_group", "O(3)")
        group_name = str(group_name)
        if group_name not in ("O(3)", "SO(3)"):
            raise NotImplementedError(f"equivariance_invariance_group={group_name!r}")
        if any(k.startswith("tensor_embedding.") and "state" in k for k in sd):
            raise NotImplementedError("State features not implemented for distributed computation.")
        units = int(sd["tensor_embedding.emb.weight"].shape[1])
        layers = sorted({int(k.split(".")[1]) for k in sd if k.startswith("layers.")})
        width = getattr(getattr(self._attr("bond_expansion"), "rbf", None), "width", None)
        if width is None:
            raise NotImplementedError("bond_expansion.rbf.width not found")
        eng = _lib.Engine(
            n_elem=int(sd["tensor_embedding.emb.weight"].shape[0]), n_blocks=len(layers), cutoff=float(self._attr("cutoff")),
            tensornet=dict(units=units, num_rbf=int(sd["bond_expansion.rbf.centers"].shape[0]),
                           so3=group_name == "SO(3)", rbf_width=float(width)),
            device=[int(g) for g in gpus] if group else int(gpus[rank]))
        self._attach_engine(eng, gpus, rank, world, group, balance)
