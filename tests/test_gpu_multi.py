"""`-m gpu` multi-GPU tests (need >= 2 visible GPUs; skipped on a single-GPU machine).  The N > 1 host logic is
covered on CPU by the gloo tests in tests/test_host_cpu.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tiled_amg_across_ranks_equals_single_process(tmp_path):
    out = str(tmp_path / "res.npz")
    n = min(4, torch.cuda.device_count())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29517", os.path.join(HERE, "dist_tiled_amg.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    assert int(z["ok"]) == 1 and int(z["n_instances"]) > 0 and int(z["world"]) == n


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_training_step_gradients(tmp_path):
    """cfg 5 across ranks: per-rank training step + NCCL all-reduce of the flat gradient buffer == the average of the per-batch
    gradients computed in one process (DDP semantics of micro_sam/training/training.py:train_sam)."""
    out = str(tmp_path / "res.npz")
    n = min(4, torch.cuda.device_count())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29519", os.path.join(HERE, "dist_train_step.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    assert int(z["ok"]) == 1 and int(z["world"]) == n and int(z["n"]) > 1_000_000, dict(z)
