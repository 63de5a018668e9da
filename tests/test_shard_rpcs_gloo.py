"""The replicated calls of RangeShardedDispatcher on CPU: two gloo ranks over the CPU checker, where every replica holds
every lease, answer KeepTaskAlive, NotifyServantRunningTasks, GetRunningTasks, the in-flight index, a window of
WaitForStartingTask RPCs and a group SchedulerService exactly as one scheduler."""
import os
import socket
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
PORT_LIB = ROOT / "oracle" / "libydoracle.so"


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _script(d, sd, svc):
    """The calls, on a RangeShardedDispatcher `sd` over `d` (or on one TaskDispatcher: sd is d)."""
    from yadcc_b200 import RunningTask, _abi
    from yadcc_b200 import streams as S
    from yadcc_b200.service import HeartbeatRequest

    w = S.config3(3000, 60, 6)
    w.register(d, now=0.0, expires_in=100.0)
    out = []
    rpcs = np.zeros(5, dtype=_abi.RPC_WAIT_DTYPE)
    for i in range(5):
        rpcs[i] = (d.intern_env(w.digests[i % len(w.digests)]), 0, d.intern_ip("172.16.0.9"), 40 * (i + 1), 10, 0,
                   10_000_000_000)
    res, gr = sd.wait_for_starting_task_rpcs(rpcs, 0.5)
    out += [res.tolist(), gr.tolist()]
    ids = gr["task_id"]
    out.append(sd.keep_tasks_alive(list(ids[::2]) + [10**9], 5.0, now=0.6).tolist())
    loc = d.servant_location(int(gr["servant_index"][0]))
    mine = [int(t) for t, s in zip(ids, gr["servant_index"]) if d.servant_location(int(s)) == loc]
    tasks = [RunningTask(k, t, loc, f"{t:064x}") for k, t in enumerate(mine + [777777])]
    out.append(sd.notify_servants_running_tasks([(loc, tasks), ("10.254.0.1:1", tasks[:1])]))
    out.append([(t.servant_task_id, t.task_grant_id, t.servant_location, t.task_digest) for t in sd.get_running_tasks()])
    out.append(sd.running_index_refresh())
    out.append(d.find_running_tasks([f"{t:064x}" for t in mine[:3]] + ["00" * 32]).tolist())
    st, tok = svc.get_config("u", now=0.7)
    out.append(st)
    hb = HeartbeatRequest(token="s", location=loc, remote_ip=loc.split(":")[0], next_heartbeat_in_ms=5000, version=9,
                          num_processors=16, capacity=8, total_memory_in_bytes=64 << 30, memory_available_in_bytes=50 << 30,
                          env_digests=list(d.servant_personality(int(gr["servant_index"][0])).environments),
                          running_tasks=tasks[:2])
    r = svc.heartbeat(hb, now=0.8)
    out.append((r.status, r.expired_tasks, r.acceptable_tokens[1] == tok))
    out.append(svc.keep_task_alive("u", [int(x) for x in ids[:4]], 3000, now=0.9)[1].tolist())
    out.append(svc.free_task("u", [int(x) for x in ids[:3]]))
    out.append([(t.task_grant_id, t.servant_location) for t in svc.get_running_tasks()])
    out.append(d.servant_state()["running_tasks"].tolist())
    return out, tok


def _rank_main(rank, world, port, out_dir):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200.service import SchedulerService
    from yadcc_b200.sharded import RangeShardedDispatcher

    d = TaskDispatcher(str(PORT_LIB))
    sd = RangeShardedDispatcher(d, rank, world)
    assert not sd.native
    svc = SchedulerService(sd, acceptable_user_tokens="u", acceptable_servant_tokens="s")  # token_seed 0
    out, tok = _script(d, sd, svc)
    np.save(Path(out_dir) / f"rank{rank}.npy", np.asarray([out, tok], dtype=object), allow_pickle=True)
    svc.close()
    dist.barrier()
    dist.destroy_process_group()


def test_replicated_calls_on_two_gloo_ranks_equal_one_scheduler(tmp_path, port_lib):
    import torch.multiprocessing as mp
    from yadcc_b200 import TaskDispatcher
    from yadcc_b200.service import SchedulerService

    world = 2
    mp.spawn(_rank_main, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    one = TaskDispatcher(port_lib)
    want, _ = _script(one, one, SchedulerService(one, acceptable_user_tokens="u", acceptable_servant_tokens="s"))
    ranks = [np.load(tmp_path / f"rank{r}.npy", allow_pickle=True) for r in range(world)]
    for r in range(world):
        assert list(ranks[r][0]) == want, r
    assert ranks[0][1] == ranks[1][1], "the ranks hand out different serving-daemon tokens"
