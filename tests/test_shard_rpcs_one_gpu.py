"""The replicated calls of the range-sharded scheduler (include/ydshard.h) on ONE GPU: W ranks as W threads of one
process over the test-only NCCL stand-in (tests/fake_nccl), every rank's answer checked against the CPU checker fed the
whole queue (tests/shard_rpcs_check.py).  Keep-alive, heartbeat notification, GetRunningTasks, the in-flight index,
windows of WaitForStartingTask RPCs, and a SchedulerServiceImpl and the wire layer over the group."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_rpcs_check.py"
FUZZ_SEEDS = [s for s in range(1, 60) if s % 5 != 0][:40]  # (the seeds of test_shard_one_gpu.py)


def _run(*args, timeout=900):
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "oracle" / "libydoracle.so",
              ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(HARNESS), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_rpcs") is True, msg
    if "--real-nccl" not in args:
        assert lines[-1]["nccl"] == "fake_nccl" and not lines[-1]["torch_loaded"], msg
    return [x for x in lines[:-1] if "case" in x and "ok" in x], msg


@pytest.mark.gpu
@pytest.mark.parametrize("unique_hosts", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_fuzz_streams(world, unique_hosts):
    args = ["--world", str(world), "--fuzz", ",".join(map(str, FUZZ_SEEDS)), "--seed", str(world)]
    cases, msg = _run(*(args + (["--unique-hosts"] if unique_hosts else [])))
    assert len(cases) == len(FUZZ_SEEDS) and all(c["ok"] for c in cases), msg
    for k in ("keepalive", "notify", "running", "index"):
        assert sum(c[k] for c in cases) > 40, (k, msg)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_rpc_windows(world):
    """Mixed immediate and prefetch counts, malformed RPCs, unknown environments on immediate and prefetch-only RPCs,
    counts above the capacity bound, windows of fewer decisions than ranks, requestors behind servant IPs (the
    sequential solver), and a cap one short of the window (refused on every rank)."""
    cases, msg = _run("--world", str(world), "--rpcs", "60", "--seed", str(20 + world))
    assert len(cases) == 1 and cases[0]["ok"] and cases[0]["rpc_windows"] == 60 and cases[0]["refusals"] > 0, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 4])
def test_service_and_wire_over_a_group(world):
    cases, msg = _run("--world", str(world), "--service", "--seed", str(30 + world))
    assert len(cases) == 1 and cases[0]["ok"] and cases[0]["wire_calls"] > 10 and cases[0]["service_ops"] > 0, msg


@pytest.mark.gpu
def test_real_nccl_one_rank():
    """One rank over the real libnccl.so.2 (PyTorch's): every new call once or more."""
    cases, msg = _run("--real-nccl", "--world", "1", "--fuzz", "3,7", "--rpcs", "8", "--service")
    assert len(cases) == 4 and all(c["ok"] for c in cases), msg
