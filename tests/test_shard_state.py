"""State handover of the range-sharded scheduler (yd_shard_export_state / yd_shard_import_state, include/ydshard.h).

GPU cases run tests/shard_state_check.py: W ranks as threads of one process on ONE GPU over the test-only NCCL
stand-in, against one scheduler fed the concatenated queue.  The CPU case runs RangeShardedDispatcher over gloo with
the port's state build, whose replicas each hold every lease."""
import json
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
HARNESS = ROOT / "tests" / "shard_state_check.py"
PORT_STATE_LIB = ROOT / "checkers" / "libydport_state.so"
FUZZ_SEEDS = [s for s in range(1, 60) if s % 5 != 0][:24]  # (the seeds test_shard_one_gpu.py uses; no wide clusters)


@pytest.fixture(scope="module")
def harness():
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", PORT_STATE_LIB, ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"

    def run(*args, timeout=1200):
        p = subprocess.run([sys.executable, str(HARNESS), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
        lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
        msg = p.stdout[-4000:] + p.stderr[-3000:]
        assert p.returncode == 0 and lines and lines[-1].get("shard_state") is True, msg
        assert not lines[-1]["torch_loaded"] and lines[-1]["fake_nccl_collectives"] > 0, msg
        return [x for x in lines[:-1] if "case" in x], msg

    return run


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_exports_match_the_single_scheduler(harness, world):
    """At every cut every rank exports the port checker's bytes, and the group plays on with the checker's decisions."""
    cases, msg = harness("--world", str(world), "--fuzz", ",".join(map(str, FUZZ_SEEDS)), "--mode", "export",
                         "--seed", str(world))
    assert len(cases) == len(FUZZ_SEEDS) and all(c["ok"] for c in cases), msg
    assert sum(c["cuts"] for c in cases) >= 4 * len(FUZZ_SEEDS) and sum(c["solves"] for c in cases) > 100, msg
    assert sum(c["zombie_cuts"] for c in cases) > 0, msg
    if world > 1:
        assert sum(c["split_lease_cuts"] for c in cases) > 0, msg
        assert sum(c["split_group_cuts"] for c in cases) > 0, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_handover_between_group_sizes(harness, world):
    """Each cut hands the export to a fresh group of 1..4 ranks or to a plain handle (yd_import_state), which plays the
    rest of the stream; a plain handle's export goes into a group at the next cut."""
    targets = [(world + k) % 5 for k in range(5)]  # every size and the plain handle, starting elsewhere per world
    cases, msg = harness("--world", str(world), "--fuzz", ",".join(map(str, FUZZ_SEEDS)), "--mode", "handover",
                         "--targets", ",".join(map(str, targets)), "--seed", str(10 + world))
    assert len(cases) == len(FUZZ_SEEDS) and all(c["ok"] for c in cases), msg
    assert sum(c["handovers"] for c in cases) >= 4 * len(FUZZ_SEEDS), msg


@pytest.mark.gpu
def test_scale_cfg2_mod_and_a_million_leases(harness):
    """cfg2-mod (100 k leases) and 1 M leases over four ranks: the group's export is a single CUDA handle's, and two
    handovers into fresh groups continue identically."""
    cases, msg = harness("--world", "4", "--scale", "cfg2-mod,1m", timeout=2400)
    assert [c["case"] for c in cases] == ["cfg2-mod", "1m"] and all(c["ok"] for c in cases), msg
    assert all(c["handovers"] == 2 for c in cases), msg
    print(msg)


@pytest.mark.gpu
def test_refusals_are_all_or_nothing(harness):
    cases, msg = harness("--world", "3", "--refusals")
    assert cases and cases[-1]["case"] == "refusals" and cases[-1]["ok"], msg


# ---- CPU: RangeShardedDispatcher over gloo, the port's state build --------------------------------------------------


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, out_dir, blob_in):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200 import streams as S
    from yadcc_b200.dispatcher import StateError
    from yadcc_b200.sharded import RangeShardedDispatcher

    w = S.config3(3000, 80, 6)
    d = TaskDispatcher(str(PORT_STATE_LIB))
    rs = RangeShardedDispatcher(d, rank, world)

    def my_range():  # (built after an import: interning makes a handle not fresh)
        full = w.build_requests(d)
        cut = [len(full) * r // world for r in range(world + 1)]
        return np.ascontiguousarray(full[cut[rank]:cut[rank + 1]])

    out = {}
    if blob_in is None:
        mine = my_range()
        w.register(d, now=0.0, expires_in=100.0)
        for rnd in range(2):
            g = rs.wait_for_starting_new_tasks(mine, 0.5 + rnd)
            rs.free_tasks(g["task_id"][g["status"] == 2][::3])
            d.on_expiration_timer(now=0.7 + rnd)
        out["blob"] = rs.export_state(now=2.0)
    else:
        blob = Path(blob_in).read_bytes()
        # all or nothing: one rank's truncated blob is refused on every rank, which all stay fresh
        try:
            rs.import_state(blob if rank != 1 else blob[:-3], now=2.0)
            out["refusal"] = 0
        except StateError as e:
            out["refusal"] = e.code
        out["fresh"] = d.num_servants() == 0 and d.next_task_id() == 0
        rs.import_state(blob, now=2.0)
        mine = my_range()
        g = rs.wait_for_starting_new_tasks(mine, 2.5)
        rs.free_tasks(g["task_id"][g["status"] == 2][::3])
        d.on_expiration_timer(now=2.7)
        out["grants"] = g
        out["blob"] = rs.export_state(now=3.0)
    np.save(Path(out_dir) / f"rank{rank}.npy", np.asarray([out], dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_range_sharded_export_and_import_over_gloo(tmp_path):
    """Two gloo ranks export what one scheduler exports; three fresh ranks import it (one rank's truncated copy is
    refused everywhere first) and continue exactly like the scheduler that never stopped."""
    import torch.multiprocessing as mp
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200 import streams as S

    if not PORT_STATE_LIB.exists():
        subprocess.check_call(["make", "-C", str(ROOT), "checkers/libydport_state.so"])
    one = TaskDispatcher(str(PORT_STATE_LIB))
    w = S.config3(3000, 80, 6)
    full = w.build_requests(one)
    w.register(one, now=0.0, expires_in=100.0)
    for rnd in range(2):
        g = one.wait_for_starting_new_tasks(full, 0.5 + rnd)
        ok = g["status"] == 2
        # every rank frees every third of its own range's grants
        ids = [g["task_id"][c0:c1][ok[c0:c1]][::3] for c0, c1 in ((0, 1500), (1500, 3000))]
        one.free_tasks(np.concatenate(ids))
        one.on_expiration_timer(now=0.7 + rnd)
    want = one.export_state(now=2.0)

    a, b = tmp_path / "two", tmp_path / "three"
    a.mkdir(), b.mkdir()
    mp.spawn(_rank_main, args=(2, _free_port(), str(a), None), nprocs=2, join=True)
    blobs = [np.load(a / f"rank{r}.npy", allow_pickle=True)[0]["blob"] for r in range(2)]
    assert blobs[0] == want and blobs[1] == want
    (tmp_path / "blob").write_bytes(want)

    mp.spawn(_rank_main, args=(3, _free_port(), str(b), str(tmp_path / "blob")), nprocs=3, join=True)
    outs = [np.load(b / f"rank{r}.npy", allow_pickle=True)[0] for r in range(3)]
    assert [o["refusal"] for o in outs] == [1, 1, 1] and all(o["fresh"] for o in outs)
    g = one.wait_for_starting_new_tasks(full, 2.5)
    cut = [0, 1000, 2000, 3000]
    ids = []
    for r in range(3):
        part, ref = outs[r]["grants"], g[cut[r]:cut[r + 1]]
        for k in ("status", "servant_index", "task_id"):
            assert (part[k] == ref[k]).all(), (r, k)
        ids.append(ref["task_id"][ref["status"] == 2][::3])
    one.free_tasks(np.concatenate(ids))
    one.on_expiration_timer(now=2.7)
    final = one.export_state(now=3.0)
    assert all(o["blob"] == final for o in outs)
    one.close()
