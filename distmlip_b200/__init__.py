"""distmlip_b200 -- H100-native (sm_90a) engine behind DistMLIP's CHGNet graph-parallel hot path.

Host-side mirror of the reference package root (DistMLIP/__init__.py:9-33): global dtype flags.
fp32 is the parity dtype; indices are int32 on the device (the reference uses int64 on the host).
"""
from __future__ import annotations

import numpy as np
import torch

float_np = np.float32
float_th = torch.float
int_np = np.int32
int_th = torch.int32

__version__ = "0.1.0"


def set_default_dtype(type_: str = "float", size: int = 32):
    """Mirror of DistMLIP.set_default_dtype (DistMLIP/__init__.py:15-33); the CUDA engine is fp32 only."""
    if type_ == "float" and size != 32:
        raise ValueError("the sm_90a engine computes in fp32 only")
    if size in (16, 32, 64):
        globals()[f"{type_}_th"] = getattr(torch, f"{type_}{size}")
        globals()[f"{type_}_np"] = getattr(np, f"{type_}{size}")
    else:
        raise ValueError("Invalid dtype size")
