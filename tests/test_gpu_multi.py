"""Multi-GPU parity (needs >= 2 H100s on one host; skipped otherwise)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_block_cyclic_cholesky_and_sharded_posterior(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + world), os.path.join(ROOT, "tests", "dist_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert "DIST_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_vfe_elbo_sharded_over_two_gpus():
    """Config-4 shaped: elbo / approximate posterior with the observation chunks sharded over 2 ranks
    and one all-reduce of the M x M accumulator."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29561", os.path.join(ROOT, "tests", "dist_vfe_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert "VFE_DIST_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
