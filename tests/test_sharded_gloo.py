"""N > 1 path on CPU: two gloo ranks, each running the CPU oracle behind the same C ABI,
must reproduce a single scheduler's answers (statuses, GLOBAL task ids, servant
locations) for the whole queue.  This exercises ShardedDispatcher's ownership routing
and its one collective (all-reduce of grant flags -> global FIFO task ids)."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
PORT_LIB = ROOT / "oracle" / "libydoracle.so"


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _workload(seed=5, n_servants=120, n_tasks=4000, n_digests=6):
    from yadcc_b200 import Servant, PRIORITY_DEDICATED, PRIORITY_USER

    rng = np.random.default_rng(seed)
    digests = [f"{i:064x}" for i in range(n_digests)]
    servants = []
    for i in range(n_servants):
        d = digests[i % n_digests]
        # digests 2k and 2k+1 sometimes share a servant: they must live on the same rank
        envs = [d] + ([digests[(i % n_digests) ^ 1]] if rng.random() < 0.3 else [])
        servants.append(Servant(f"10.7.{i >> 8}.{i & 255}:8335", None, envs, int(rng.choice([7, 8])), 16,
                                int(rng.integers(0, 8)), 0, 64 << 30, int(rng.integers(0, 10)),
                                PRIORITY_DEDICATED if i % 9 == 0 else PRIORITY_USER))
    req_digest = rng.integers(0, n_digests + 1, n_tasks)  # n_digests == "nobody has it"
    req_ip = rng.integers(0, n_servants + 40, n_tasks)
    req_mv = rng.choice([7, 8], n_tasks)
    return digests, servants, req_digest, req_ip, req_mv


def _ip(j, n_servants):
    return f"10.7.{j >> 8}.{j & 255}" if j < n_servants else f"172.16.1.{j - n_servants}"


def _owner(digest: str, world: int) -> int:
    return (int(digest, 16) // 2) % world  # pairs (2k, 2k+1) stay together


def _rank_main(rank, world, port, out_dir, id_mode):
    import torch
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200.sharded import ShardedDispatcher

    digests, servants, req_digest, req_ip, req_mv = _workload()
    strided = id_mode == "strided"
    d = TaskDispatcher(str(PORT_LIB), id_stride=world if strided else 0, id_offset=rank if strided else 0)
    sd = ShardedDispatcher(d, rank, world, device=torch.device("cpu"), digest_owner=_owner, id_mode=id_mode)
    for sv in servants:
        sd.keep_servant_alive(sv, 10.0, now=0.0)
    owners = np.asarray([_owner(digests[k], world) if k < len(digests) else -1 for k in req_digest])
    mine = np.nonzero(owners == rank)[0]
    all_d = digests + ["ff" * 32]
    results = []
    for rnd in range(2):  # two solves: the second one continues the global id space
        reqs = d.make_requests(len(mine), [all_d[req_digest[i]] for i in mine],
                               [_ip(int(req_ip[i]), len(servants)) for i in mine], req_mv[mine].astype(np.uint32))
        g = sd.wait_for_starting_new_tasks(None, owners, reqs, now=0.5 + rnd)
        loc = np.asarray([d.servant_location(int(x)) or "" for x in g["servant_index"]])
        results.append((mine, g["status"].copy(), g["task_id"].copy(), loc))
        # free every third grant through the GLOBAL ids, then renew the rest
        ok = g["status"] == 2
        sd.free_tasks(g["task_id"][ok][::3])
        if strided:  # ids of the other shard are ignored, not mistaken for local ones
            foreign = g["task_id"][ok][1::3] - np.uint64(rank) + np.uint64((rank + 1) % world)
            assert not sd.keep_tasks_alive(foreign, 5.0, now=0.6 + rnd).any()
            sd.free_tasks(foreign)
            assert sd.keep_tasks_alive(g["task_id"][ok][1::3], 5.0, now=0.6 + rnd).all()
    np.save(Path(out_dir) / f"rank{rank}.npy", np.asarray(results, dtype=object), allow_pickle=True)
    assert (sd.collective_bytes > 0) == (id_mode == "fifo")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("id_mode", ["fifo", "strided"])
def test_two_ranks_equal_one_scheduler(tmp_path, port_lib, id_mode):
    import torch.multiprocessing as mp
    from yadcc_b200 import TaskDispatcher

    world = 2
    mp.spawn(_rank_main, args=(world, _free_port(), str(tmp_path), id_mode), nprocs=world, join=True)

    digests, servants, req_digest, req_ip, req_mv = _workload()
    one = TaskDispatcher(port_lib)
    for sv in servants:
        one.keep_servant_alive(sv, 10.0, now=0.0)
    all_d = digests + ["ff" * 32]
    ranks = [np.load(tmp_path / f"rank{r}.npy", allow_pickle=True) for r in range(world)]
    for rnd in range(2):
        reqs = one.make_requests(len(req_digest), [all_d[k] for k in req_digest],
                                 [_ip(int(j), len(servants)) for j in req_ip], req_mv.astype(np.uint32))
        g = one.wait_for_starting_new_tasks(reqs, 0.5 + rnd)
        loc = np.asarray([one.servant_location(int(x)) or "" for x in g["servant_index"]])
        seen = np.zeros(len(g), dtype=bool)
        for r in range(world):
            mine, status, task_id, rloc = ranks[r][rnd]
            mine = np.asarray(mine, dtype=np.int64)
            status, task_id = np.asarray(status, dtype=np.uint32), np.asarray(task_id, dtype=np.uint64)
            rloc = np.asarray(rloc, dtype=str)
            seen[mine] = True
            assert (status == g["status"][mine]).all()
            ok = status == 2
            if id_mode == "fifo":
                assert (task_id[ok] == g["task_id"][mine][ok]).all(), "global task ids"
            else:  # local FIFO number * world + rank: unique, routable, in the shard's own grant order
                assert (task_id[ok] % world == r).all()
                local = task_id[ok] // world
                assert (np.diff(local.astype(np.int64)) == 1).all() and (rnd > 0 or local[0] == 0)
            assert (rloc[ok] == loc[mine][ok]).all()
        # requests nobody owns are exactly the unknown-digest ones: EnvironmentNotFound
        assert (g["status"][~seen] == 0).all()
        # mirror the per-rank "free every third of MY grants"
        for r in range(world):
            mine, status, task_id, _ = ranks[r][rnd]
            mine = np.asarray(mine, dtype=np.int64)
            status, task_id = np.asarray(status, dtype=np.uint32), np.asarray(task_id, dtype=np.uint64)
            if id_mode == "fifo":
                one.free_tasks(task_id[status == 2][::3])
            else:  # the same requests' grants in the single scheduler's numbering
                one.free_tasks(g["task_id"][mine][status == 2][::3])


def _range_rank_main(rank, world, port, out_dir):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200 import streams as S
    from yadcc_b200.sharded import RangeShardedDispatcher

    w = S.config3(6000, 120, 6)
    d = TaskDispatcher(str(PORT_LIB))
    w.register(d, now=0.0, expires_in=100.0)  # replicated servant table: every rank hears every heartbeat
    full = w.build_requests(d)
    cut = [0, 1700, len(full)]  # uneven contiguous ranges of ONE FIFO queue
    mine = np.ascontiguousarray(full[cut[rank]:cut[rank + 1]])
    sd = RangeShardedDispatcher(d, rank, world)
    out = []
    for rnd in range(2):
        g = sd.wait_for_starting_new_tasks(mine, 0.5 + rnd)
        out.append(g.copy())
        ok = g["status"] == 2
        sd.free_tasks(g["task_id"][ok][rank::3])  # collective: every rank names some of ITS grants
        d.on_expiration_timer(now=0.7 + rnd)
    st = d.servant_state()
    np.save(Path(out_dir) / f"range{rank}.npy", np.asarray([out[0], out[1], st], dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_range_sharded_queue_on_two_gloo_ranks_equals_one_scheduler(tmp_path, port_lib):
    """The range-sharded scheduler's contract (include/ydshard.h) on CPU: two gloo ranks, each with its contiguous
    range of one FIFO queue and a replica of the servant table, make together exactly the decisions -- statuses,
    servants, FIFO task ids, per-servant bookkeeping -- of one TaskDispatcher fed the whole queue, across a
    collective FreeTask.  (On GPUs the exchange is the C++/NCCL path; tests/multi_gpu_check.py checks that one.)"""
    import torch.multiprocessing as mp
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200 import streams as S

    world = 2
    mp.spawn(_range_rank_main, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    w = S.config3(6000, 120, 6)
    one = TaskDispatcher(port_lib)
    w.register(one, now=0.0, expires_in=100.0)
    full = w.build_requests(one)
    cut = [0, 1700, len(full)]
    ranks = [np.load(tmp_path / f"range{r}.npy", allow_pickle=True) for r in range(world)]
    for rnd in range(2):
        g = one.wait_for_starting_new_tasks(full, 0.5 + rnd)
        for r in range(world):
            part = ranks[r][rnd]
            ref = g[cut[r]:cut[r + 1]]
            for k in ("status", "servant_index", "task_id"):
                assert (np.asarray(part[k]) == ref[k]).all(), (rnd, r, k)
            ok = ref["status"] == 2
            one.free_tasks(ref["task_id"][ok][r::3])
        one.on_expiration_timer(now=0.7 + rnd)
    st = one.servant_state()
    for r in range(world):
        assert (np.asarray(ranks[r][2]["running_tasks"]) == st["running_tasks"]).all()


def test_component_digest_owner_keeps_components_together():
    """ADVICE (round 1): with the plain crc32 map a servant advertising two compilers usually has its digests on
    different ranks; the component-aware map derives ownership from the connected components."""
    from yadcc_b200 import Servant
    from yadcc_b200.sharded import ShardedDispatcher, component_digest_owner, default_digest_owner

    digs = [f"{i:02x}" * 32 for i in range(12)]
    servants = [Servant(f"10.0.0.{i}:1", None, [digs[i % 12], digs[(i * 5 + 1) % 12]] if i % 3 else [digs[i % 12]], 1, 8, 0, 0, 0, 8)
                for i in range(40)]
    servants.append(Servant("10.0.1.1:1", None, [], 1, 8, 0, 0, 0, 8))
    world = 4
    owner = component_digest_owner(servants, world)
    for sv in servants:
        assert len({owner(d, world) for d in sv.environments}) <= 1
    assert owner("ff" * 32, world) == default_digest_owner("ff" * 32, world)  # a digest nobody holds
    # the plain map does split at least one of these servants (that is what the helper is for)
    assert any(len({default_digest_owner(d, world) for d in sv.environments}) > 1 for sv in servants)
    sd = ShardedDispatcher.__new__(ShardedDispatcher)
    sd.world, sd.digest_owner = world, owner
    for sv in servants:
        sd.owner_of_servant(sv)  # does not raise
