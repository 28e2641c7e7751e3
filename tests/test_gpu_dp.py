"""Row (e) on real GPUs: two ranks, per-rank env shards, gradients all-reduced by the in-library NCCL communicator inside
the captured training graph; equal to one GPU training on the concatenated rollout.  Skips on a single-GPU box (the
scaling identity it rests on is checked on the CPU by test_oracle_golden.py::test_data_parallel_gradient_identity)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_rank_data_parallel_equals_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "tools", "dp_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=ROOT)
    assert res.returncode == 0 and "DP_CHECK_OK" in res.stdout, (res.stdout[-1500:], res.stderr[-1500:])
