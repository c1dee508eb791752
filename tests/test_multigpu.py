"""Data-parallel path across REAL ranks (one process per GPU, NCCL over NVLink): needs >= 2 visible GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_pipeline_is_shard_invariant_across_two_ranks():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = str(29600 + os.getpid() % 300)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", port, os.path.join(REPO, "tests", "_mgpu_worker.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MGPU_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-3000:])
