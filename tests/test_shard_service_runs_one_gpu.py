"""Runs of Heartbeat, KeepTaskAlive and FreeTask frames on a range-sharded group's services: W = 1..4 ranks as threads of
one process over the test-only NCCL stand-in, every rank's bytes checked against one service over the CPU checker fed
the frames one by one, a run's collectives checked not to grow with its length, and yd_shard_keep_tasks_alive checked
against the checker (tests/shard_service_runs_check.py)."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_service_runs_check.py"


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_group_service_runs(world):
    pytest.importorskip("google.protobuf")
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "checkers" / "libydport_state.so",
              ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(HARNESS), "--world", str(world)], capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_service_runs") is True, msg
    assert not lines[-1]["torch_loaded"], msg
    cases = {c["case"]: c for c in lines[:-1]}
    assert cases["streams"]["frames"] > 300, msg
    assert cases["keep_tasks_alive"]["calls"] == 5, msg
    per_run = cases["collectives"]["per_run"]
    assert sorted(per_run) == ["FreeTask", "Heartbeat", "KeepTaskAlive"], msg
