"""The pre-filtered solve of RangeShardedDispatcher on CPU: two gloo ranks over the CPU checker with the task keys
(checkers/libydport_keys.so), each passing its own range (and, for descriptors, its own argument table), get exactly
their slice of what one scheduler's single-handle call returns for the concatenated queue."""
import os
import pickle
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
KEYS_LIB = ROOT / "checkers" / "libydport_keys.so"
WORLD = 2
CUTS = {"keys": [0, 300, 700], "desc": [0, 0, 500], "desc2": [0, 450, 800]}  # (the second: rank 0's range empty)


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _cluster(d):
    """The same state on every replica: servants, a bloom filter with some cache keys, leases reported as running
    with their task digests and the in-flight index refreshed from them.  Returns the request queue and per-request
    (argument string, source digest) descriptors."""
    from yadcc_b200 import TaskSources, _abi
    from yadcc_b200 import streams as S
    from yadcc_b200.dispatcher import RunningTask

    w = S.config3(2400, 40, 4)
    w.register(d, now=0.0, expires_in=100.0)
    reqs = w.build_requests(d)
    rng = np.random.default_rng(5)
    args = [bytes(rng.integers(32, 127, int(m), dtype=np.uint8)) for m in np.geomspace(30, 2500, 9).astype(int)]
    tu = rng.integers(0, 150, len(reqs))  # 150 translation units: repeated tasks
    tu_args = rng.integers(0, len(args), 150)[tu]
    tu_src = np.frombuffer(rng.bytes(32 * 150), dtype=np.uint8).reshape(150, 32)[tu]
    src = TaskSources.of(args, tu_args, tu_src)
    keys, digests = d.derive_task_keys(reqs, src)
    d.bloom_reset(1 << 16, 4)
    d.bloom_add(keys[:300:4])
    g = d.wait_for_starting_new_tasks(reqs[:300].copy(), 0.5)
    by: dict = {}
    for j, x in enumerate(g.tolist()):
        if x[2] == _abi.STATUS_GRANTED:
            by.setdefault(x[1], []).append(RunningTask(j + 1, x[0], d.servant_location(x[1]), bytes(digests[j]).decode()))
    d.notify_servants_running_tasks([(d.servant_location(k), v) for k, v in by.items()])
    d.running_index_refresh()
    return reqs[300:], args, tu_args[300:], tu_src[300:]


def _rank_sources(args, tu_args, tu_src, lo, hi, rank):
    """This rank's own argument table (the strings in a rank-specific order) for requests [lo, hi)."""
    from yadcc_b200 import TaskSources

    order = list(range(len(args)))[::-1] if rank % 2 else list(range(len(args)))
    pos = {a: k for k, a in enumerate(order)}
    return TaskSources.of([args[a] for a in order], np.asarray([pos[int(a)] for a in tu_args[lo:hi]], dtype=np.uint32),
                          tu_src[lo:hi])


def _rank_main(rank, world, port, out_dir):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yadcc_b200 import TaskDispatcher, TaskKeysError, TaskSources
    from yadcc_b200.sharded import RangeShardedDispatcher

    d = TaskDispatcher(str(KEYS_LIB))
    sd = RangeShardedDispatcher(d, rank, world)
    assert not sd.native
    q, args, tu_args, tu_src = _cluster(d)
    out = []
    lo, hi = CUTS["keys"][rank], CUTS["keys"][rank + 1]
    keys, digests = d.derive_task_keys(q[:700].copy(), TaskSources.of(args, tu_args[:700], tu_src[:700]))
    out.append(sd.filter_and_wait_for_starting_new_tasks(q[lo:hi].copy(), keys[lo:hi], digests[lo:hi], 1.0))
    out.append(sd.filter_and_wait_for_starting_new_tasks(q[lo:hi].copy(), None, digests[lo:hi], 1.1))
    for name, base, stages, t in (("desc", 700, 3, 1.2), ("desc2", 1200, 1, 1.3)):
        lo, hi = base + CUTS[name][rank], base + CUTS[name][rank + 1]
        out.append(sd.derive_filter_and_wait_for_starting_new_tasks(q[lo:hi].copy(), _rank_sources(args, tu_args, tu_src, lo, hi, rank),
                                                                    stages, t))
    # rank 1's descriptors refused: every rank raises, rank 1 with its own code, and nothing is decided
    lo, hi = 1800 + 100 * rank, 1900 + 100 * rank
    bad = _rank_sources(args, tu_args, tu_src, lo, hi, rank)
    if rank == 1:
        bad.args_index[3] = 99
    try:
        sd.derive_filter_and_wait_for_starting_new_tasks(q[lo:hi].copy(), bad, 3, 1.4)
        out.append("decided")
    except TaskKeysError as e:
        out.append(("TaskKeysError", e.code))
    except RuntimeError:
        out.append("RuntimeError")
    out.append((d.next_task_id(), d.servant_state()["running_tasks"].tolist()))
    (Path(out_dir) / f"rank{rank}.pkl").write_bytes(pickle.dumps(out))
    dist.barrier()
    dist.destroy_process_group()


def _slice(whole, lo, hi):
    v, h, g = whole
    first = int((v[:lo] == 0).sum())
    mine = int((v[lo:hi] == 0).sum())
    return v[lo:hi], h[lo:hi], g[first:first + mine]


def test_filter_calls_on_two_gloo_ranks_equal_one_scheduler(tmp_path):
    import torch.multiprocessing as mp
    from yadcc_b200 import TaskDispatcher, TaskSources

    if not KEYS_LIB.exists():
        subprocess.check_call(["make", "-C", str(ROOT), "checkers/libydport_keys.so"])
    mp.spawn(_rank_main, args=(WORLD, _free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    one = TaskDispatcher(str(KEYS_LIB))
    q, args, tu_args, tu_src = _cluster(one)
    keys, digests = one.derive_task_keys(q[:700].copy(), TaskSources.of(args, tu_args[:700], tu_src[:700]))
    want = [one.filter_and_wait_for_starting_new_tasks(q[:700].copy(), keys, digests, 1.0),
            one.filter_and_wait_for_starting_new_tasks(q[:700].copy(), None, digests, 1.1)]
    cuts = [CUTS["keys"], CUTS["keys"]]
    for name, base, stages, t in (("desc", 700, 3, 1.2), ("desc2", 1200, 1, 1.3)):
        c = CUTS[name]
        srcs = [_rank_sources(args, tu_args, tu_src, base + c[r], base + c[r + 1], r) for r in range(WORLD)]
        whole = TaskSources.concat(srcs, [c[r + 1] - c[r] for r in range(WORLD)])
        want.append(one.derive_filter_and_wait_for_starting_new_tasks(q[base:base + c[-1]].copy(), whole, stages, t))
        cuts.append(c)
    ranks = [pickle.loads((tmp_path / f"rank{r}.pkl").read_bytes()) for r in range(WORLD)]
    verdicts = np.concatenate([w[0] for w in want])
    assert (verdicts == 1).any() and (verdicts == 2).any() and (verdicts == 0).any()  # every verdict occurs
    for r in range(WORLD):
        for k, (w, c) in enumerate(zip(want, cuts)):
            got = ranks[r][k]
            exp = _slice(w, c[r], c[r + 1])
            for a, b in zip(got, exp):
                assert a.dtype == b.dtype and a.tolist() == b.tolist(), (r, k)
    assert ranks[0][4] == "RuntimeError" and ranks[1][4] == ("TaskKeysError", 3)
    state = (one.next_task_id(), one.servant_state()["running_tasks"].tolist())
    assert ranks[0][5] == state and ranks[1][5] == state
