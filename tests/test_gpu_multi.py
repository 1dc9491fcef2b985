"""Multi-GPU checks (need >= 2 H100s on the box; skipped on a single-GPU box): the sharded forward with every
exchange mode -- NCCL collectives and the fused P2P / multicast epilogue -- is bit-identical to the single-GPU forward."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least 2 GPUs")
def test_sharded_forward_matches_single_gpu_on_all_exchanges():
    n = min(torch.cuda.device_count(), 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "scripts", "dist_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("bit-exact=True") >= 5 * n and "bit-exact=False" not in out.stdout
