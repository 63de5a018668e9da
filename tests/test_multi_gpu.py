"""The range-sharded scheduler (include/ydshard.h) on real GPUs: launches tests/multi_gpu_check.py under
torchrun with every visible GPU (>= 2) and requires its verdict.  The script compares every decision
with ONE scheduler fed the whole queue and cfg5-1m with the reference's digest."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.gpu
def test_range_sharded_queue_equals_one_scheduler():
    import torch

    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    world = 2 if n < 4 else 4
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29517", str(ROOT / "tests" / "multi_gpu_check.py"), "--quick"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    assert p.returncode == 0 and lines and lines[-1].get("multi_gpu_parity") is True, p.stdout[-3000:] + p.stderr[-3000:]
