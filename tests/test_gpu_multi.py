"""N > 1 on real GPUs: sharded run + end-of-frame gather == monolithic oracle (SURVEY.md §8(e), BASELINE.json configs[4] layout)."""

import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def test_two_gpu_sharded_gather_matches_monolithic_oracle(cuda_lib, oracle_lib):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29611", os.path.join(root, "tests", "mp_peer_gather_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "MULTI_GPU_OK world=2" in out.stdout
