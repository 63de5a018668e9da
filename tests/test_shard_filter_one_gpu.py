"""The pre-filtered solve of a range-sharded group (yd_shard_filter_and_wait_for_starting_new_tasks,
yd_shard_derive_filter_and_wait_for_starting_new_tasks) on ONE GPU: W ranks as W threads of one process over the
test-only NCCL stand-in (tests/fake_nccl), every rank's verdicts, hits, offered count and grants checked exactly against
one CPU checker handle fed the concatenated queue, and the replicas' running_tasks and next task id after every call
(tests/shard_filter_check.py)."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_filter_check.py"


def _run(*args, timeout=900):
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "checkers" / "libydport_keys.so",
              ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(HARNESS), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_filter") is True, msg
    if "--real-nccl" not in args:
        assert lines[-1]["nccl"] == "fake_nccl" and not lines[-1]["torch_loaded"], msg
    return [x for x in lines[:-1] if "case" in x and "ok" in x], msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_filter_calls_equal_one_scheduler(world):
    """Keys and descriptors, each with the stage sets none, cache, dedupe and both; random cuts with empty ranges, a
    range filtered out entirely, everything filtered out, JOINED hits on leases another rank holds, batches the
    sequential solver decides (requestors behind servant IPs), one rank's descriptors refused, and the staged offered
    queue decided again after every call."""
    calls = 8
    cases, msg = _run("--world", str(world), "--fuzz", str(calls), "--seed", str(world))
    assert len(cases) == 1 and cases[0]["ok"], msg
    c = cases[0]
    assert c["calls"] == 2 * 4 * calls and c["redecided"] == c["calls"], msg
    for k in ("offered", "cache_hits", "joined", "all_filtered", "handbacks", "refusals"):
        assert c[k] > 0, (k, msg)
    if world > 1:
        for k in ("empty_ranges", "filtered_ranges", "joined_across"):
            assert c[k] > 0, (k, msg)


@pytest.mark.gpu
def test_configs3_descriptor_queue_over_four_ranks():
    cases, msg = _run("--world", "4", "--config3", "--seed", "5")
    assert len(cases) == 1 and cases[0]["ok"] and cases[0]["calls"] == 2, msg
    assert cases[0]["cache_hits"] > 0 and cases[0]["joined"] > 0, msg


@pytest.mark.gpu
def test_real_nccl_one_rank():
    """One rank over the real libnccl.so.2 (PyTorch's)."""
    cases, msg = _run("--real-nccl", "--world", "1", "--fuzz", "3", "--seed", "9")
    assert len(cases) == 1 and cases[0]["ok"], msg
