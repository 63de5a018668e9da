"""The packed solve of a range-sharded group (yd_shard_wait_for_starting_new_tasks_packed, include/ydshard.h): 16-byte
requests up and 8-byte grants down on every rank.  On the GPU, W ranks run as W threads of one process over the test-only
NCCL stand-in (tests/shard_packed_check.py): every packed solve is checked bit for bit against one CPU checker fed the
concatenated queue through its own packed call, and against an unpacked twin group fed the same events."""
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest

from conftest import CUDA_LIB
from yadcc_b200 import _abi

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_packed_check.py"
FUZZ_SEEDS = [s for s in range(1, 40) if s % 5 != 0][:16]  # (fuzz seeds that are multiples of 5 are the wide ones)


def _run(*args, env=None, timeout=900):
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "oracle" / "libydoracle.so", Path(CUDA_LIB)):
        assert p.exists(), f"{p} missing: run build()"
    e = dict(os.environ)
    e.update(env or {})
    p = subprocess.run([sys.executable, str(HARNESS), *args], capture_output=True, text=True, timeout=timeout, env=e,
                       cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_packed") is True, msg
    if "--real-nccl" not in args:
        assert lines[-1]["nccl"] == "fake_nccl" and not lines[-1]["torch_loaded"], msg
    return [x for x in lines[:-1] if "case" in x and "ok" in x], p.stderr, msg


def test_shard_prototypes_cover_header():
    """Every function include/ydshard.h declares is in _abi's list, which load_library() requires of the CUDA library."""
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "ydshard.h").read_text(), flags=re.S)
    declared = sorted(set(re.findall(r"\b(yd_shard_[a-z_]+)\s*\(", text)))
    assert "yd_shard_wait_for_starting_new_tasks_packed" in declared
    assert declared == sorted(name for name, _, _ in _abi.SHARD_PROTOTYPES)
    lib = _abi.load_library()  # (the product library: a missing ydshard.h symbol raises AttributeError)
    assert lib.yd_shard_wait_for_starting_new_tasks_packed.argtypes is not None


@pytest.mark.gpu
@pytest.mark.parametrize("unique_hosts", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_packed_equals_checker_and_unpacked_twin(world, unique_hosts):
    """Seeded streams with even, uneven, empty and one-request ranges; packed solves interleaved with unpacked ones, frees
    of packed-granted ids, keep-alives, heartbeats and ticks; staged ranges; the whole-queue fallback (several servants
    behind one IP)."""
    args = ["--world", str(world), "--fuzz", ",".join(map(str, FUZZ_SEEDS)), "--seed", str(world)]
    cases, _, msg = _run(*(args + (["--unique-hosts"] if unique_hosts else [])))
    assert len(cases) == len(FUZZ_SEEDS) and all(c["ok"] and c["twin"] for c in cases), msg
    total = lambda k: sum(c.get(k, 0) for c in cases)  # noqa: E731
    assert total("packed") > 200 and total("unpacked") > 50 and total("frees") > 50, msg
    assert total("twin_equal_packed") == total("packed") and total("packed_granted") > 500, msg
    assert total("packed_staged_ranks") > 0, msg
    if not unique_hosts:
        assert total("packed_handbacks") > 0, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_packed_configs(world):
    """Two rounds of cfg2-mod-small, cfg2-random-small, cfg-self-small and cfg2-mod (100 k) with collective frees; the
    class-bound retry (48 classes) and more than 256 classes (the whole-queue fallback)."""
    names = ["cfg2-mod-small", "cfg2-random-small", "cfg-self-small", "cfg2-mod", "class-bound", "many-classes"]
    cases, _, msg = _run("--world", str(world), "--config", ",".join(names), "--seed", str(20 + world))
    assert [c["case"] for c in cases] == names and all(c["ok"] for c in cases), msg
    by = {c["case"]: c for c in cases}
    assert by["class-bound"]["retried"] >= 1, msg
    assert by["many-classes"]["handbacks"] >= 1, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3])
def test_packed_leases_and_prefetch(world):
    """YD_LEASE_PREFETCH, leases of 0, 1, 2, 29 999, 30 000, 30 001 and 2^31 - 1 ms: a tick 1 ms before each expiry keeps
    the leases and one 1 ms after sweeps them, on every rank as on the checker."""
    cases, _, msg = _run("--world", str(world), "--config", "lease", "--seed", "4")
    assert len(cases) == 1 and cases[0]["ok"] and cases[0]["packed"] == 1 and cases[0]["packed_granted"] > 0, msg


@pytest.mark.gpu
def test_packed_whole_queue_fallback_debug_line():
    """Batches with several servants behind one requestor IP: every rank's YDSCHED_DEBUG line reports the whole-queue
    path, and the packed answers still equal the checker's."""
    world = 3
    cases, err, msg = _run("--world", str(world), "--config", "fallback", "--seed", "6", env={"YDSCHED_DEBUG": "1"})
    assert len(cases) == 1 and cases[0]["ok"] and cases[0]["packed_handbacks"] > 0, msg
    lines = re.findall(r"ydsched: shard rank \d+ whole queue n \d+", err)
    assert len(lines) == world * cases[0]["packed_handbacks"], (len(lines), msg)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_packed_refusals(world):
    """Not in a group, n_local above the staged count, a wide cluster, and a group queue above the packed limit (lowered
    for the test) made of ranges that each stay below it: 1 on every rank, no grant written, no state changed."""
    cases, _, msg = _run("--world", str(world), "--refusals", env={"YDSCHED_SHARD_PACKED_MAX_N": "3000"})
    assert len(cases) == 1 and cases[0]["ok"], msg
    c = cases[0]
    assert c["not_in_group"] and c["staged_count"] and c["group_limit"] and c["wide"], msg


@pytest.mark.gpu
def test_packed_real_nccl_one_rank():
    """One rank over the real libnccl.so.2 (PyTorch's): the packed call binds to it and agrees with the checker."""
    cases, _, msg = _run("--real-nccl", "--world", "1", "--fuzz", "1,2,3", "--seed", "9")
    assert len(cases) == 3 and all(c["ok"] and c["packed"] > 0 for c in cases), msg
