"""The range-sharded scheduler (include/ydshard.h) on ONE GPU: W ranks as W threads of one process, talking through
the test-only NCCL stand-in (tests/fake_nccl), each call checked against the CPU checker fed the whole queue
(tests/shard_threads_check.py).  This runs every sharded call -- solve, collective free, the class-bound retry of the
attempt loop, the batches the sequential solver decides -- without a second GPU."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_threads_check.py"
FUZZ_SEEDS = [s for s in range(1, 60) if s % 5 != 0][:40]  # (fuzz seeds that are multiples of 5 are the wide ones)


@pytest.fixture(scope="module")
def harness():
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "oracle" / "libydoracle.so",
              ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"

    def run(*args, env=None, timeout=900):
        e = dict(os.environ)
        e.update(env or {})
        p = subprocess.run([sys.executable, str(HARNESS), *args], capture_output=True, text=True, timeout=timeout, env=e,
                           cwd=ROOT)
        lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
        msg = p.stdout[-4000:] + p.stderr[-3000:]
        assert p.returncode == 0 and lines and lines[-1].get("shard_parity") is True, msg
        final = lines[-1]
        if "--real-nccl" not in args:
            assert final["nccl"] == "fake_nccl" and not final["torch_loaded"], msg
            assert final["fake_nccl_collectives"] > 0 or "--refusals" in args, msg
        return [x for x in lines[:-1] if "case" in x and "ok" in x], msg

    return run


@pytest.mark.gpu
@pytest.mark.parametrize("unique_hosts", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_fuzz_streams(harness, world, unique_hosts):
    """Zombie sweeps, servant expiry, frees of unknown and duplicate ids, several servants behind one IP (batches the
    sequential solver decides), cut points that leave ranks empty."""
    args = ["--world", str(world), "--fuzz", ",".join(map(str, FUZZ_SEEDS)), "--seed", str(world)]
    cases, msg = harness(*(args + (["--unique-hosts"] if unique_hosts else [])))
    assert len(cases) == len(FUZZ_SEEDS) and all(c["ok"] for c in cases), msg
    assert sum(c["solves"] for c in cases) > 500 and sum(c["frees"] for c in cases) > 100, msg
    if world > 1:
        assert sum(c["lazy_checks"] for c in cases) > 0, msg
    if not unique_hosts:
        assert sum(c["handbacks"] for c in cases) > 0, msg  # several ports on one IP


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_configs_two_rounds(harness, world):
    names = ["cfg2-mod-small", "cfg2-random-small", "cfg-self-small", "cfg3-20k", "cfg2-mod", "cfg2-random", "cfg-self"]
    cases, msg = harness("--world", str(world), "--config", ",".join(names), "--seed", str(10 + world))
    assert [c["case"] for c in cases] == names and all(c["ok"] for c in cases), msg
    assert all(c["solves"] == 2 and c["frees"] == 2 for c in cases), msg


@pytest.mark.gpu
def test_cfg5_1m_against_reference_digest(harness):
    cases, msg = harness("--world", "4", "--golden", timeout=1200)
    assert cases and cases[-1]["case"] == "cfg5-1m" and cases[-1]["reference_digest_equal"], msg


@pytest.mark.gpu
def test_retry_grows_class_bound(harness):
    """48 (digest, min_version) classes overflow the first class bound: the attempt loop grows it and solves again."""
    cases, msg = harness("--world", "3", "--config", "class-bound")
    assert cases[0]["ok"] and cases[0]["retried"] >= 1, msg


@pytest.mark.gpu
def test_small_merge_chunks(harness):
    """32-request merge chunks and two merge rounds: many more chunks per merge, the same decisions."""
    cases, msg = harness("--world", "2", "--config", "cfg2-random-small,cfg-self-small",
                         env={"YDSCHED_MERGE_CHUNK": "32", "YDSCHED_MERGE_ROUNDS": "2"})
    assert len(cases) == 2 and all(c["ok"] for c in cases), msg


@pytest.mark.gpu
def test_refusals(harness):
    cases, msg = harness("--world", "3", "--refusals")
    assert cases and cases[-1]["case"] == "refusals" and cases[-1]["ok"], msg


@pytest.mark.gpu
def test_real_nccl_one_rank(harness):
    """One rank over the real libnccl.so.2 (PyTorch's): the library's binding to NCCL itself."""
    cases, msg = harness("--real-nccl", "--world", "1", "--fuzz", "3,7", "--config", "cfg2-mod-small")
    assert len(cases) == 3 and all(c["ok"] for c in cases), msg
