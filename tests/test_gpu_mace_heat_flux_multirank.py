"""MACE heat flux with one process per GPU (NCCL): only runs where at least two H100s are visible (skipped with one
GPU)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_rank_mace_heat_flux():
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", "29551",
           os.path.join(ROOT, "tests", "run_mace_heat_flux_multirank.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "MACE HEAT FLUX MULTIRANK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
