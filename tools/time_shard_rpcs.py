#!/usr/bin/env python
"""Host time of the range-sharded group's replicated calls (include/ydshard.h) at W ranks.

The ranks are threads of one process on ONE GPU over the test-only NCCL stand-in (tests/fake_nccl, as in
tests/shard_rpcs_check.py), so the times include the stand-in's host copies and say nothing about NVLink exchange time.
Every call ends in a device synchronise; per call the host wall-clock of the slowest rank, median of `--reps`.  Loads:
cfg2-mod's servants (2 k, 64 slots each) with 100 k leases granted by one sharded solve; keep-alive of 10 k ids; a
notification of 2 k heartbeats x 50 tasks; GetRunningTasks with the 100 k reported tasks; and a window of cfg2-mod's
100 k requests as one-decision RPCs, each decided on a fresh group.  One JSON line with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE = C.CDLL(str(ROOT / "tests" / "fake_nccl" / "libnccl.so.2"), mode=C.RTLD_GLOBAL)  # before anything loads NCCL

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT_DTYPE, RPC_WAIT_DTYPE  # noqa: E402
from yadcc_b200.dispatcher import RunningTask, TaskDispatcher  # noqa: E402


def par(fns):
    import threading

    out = [None] * len(fns)
    ts = [threading.Thread(target=lambda i=i, f=f: out.__setitem__(i, f())) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def group(lib, world, w):
    ranks = [TaskDispatcher(lib) for _ in range(world)]
    uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
    assert lib.yd_shard_unique_id(uid) == 0
    assert par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, world, uid) for r in range(world)]) == [0] * world
    for d in ranks:
        w.register(d, now=0.0, expires_in=3600.0)
    return ranks


def close(lib, ranks):
    for d in ranks:
        lib.yd_shard_finalize(d._h)
        d.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    W = a.world
    lib = _abi.load_library()
    w = S.config2(variant="mod")
    out = {"world": W, "nccl": "fake_nccl (threads on one GPU)", "reps": a.reps}

    def median_slowest(per_rank_fns, reps=a.reps, before=None):
        ts = []
        for _ in range(reps):
            if before:
                before()
            ts.append(max(par([lambda f=f: timed(f) for f in per_rank_fns])))
        return round(float(np.median(ts)), 3)

    # 100 k leases from one sharded solve
    ranks = group(lib, W, w)
    full = w.build_requests(ranks[0])
    n = len(full)
    cuts = [n * g // W for g in range(W + 1)]
    parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(W)]
    outs = [np.zeros(max(len(p), 1), dtype=GRANT_DTYPE) for p in parts]
    assert par([lambda r=r: lib.yd_shard_wait_for_starting_new_tasks(ranks[r]._h, 1_000_000, parts[r].ctypes.data,
                                                                      len(parts[r]), outs[r].ctypes.data)
                for r in range(W)]) == [0] * W
    g = np.concatenate([outs[r][:len(parts[r])] for r in range(W)])
    ok = g["status"] == _abi.STATUS_GRANTED
    ids, srv = g["task_id"][ok], g["servant_index"][ok]
    out["leases"] = int(ok.sum())

    ka = np.ascontiguousarray(ids[:10_000])
    out["keep_alive_10k_ms"] = median_slowest(
        [lambda d=d: d._keep_alive_with(lib.yd_shard_keep_task_alive, ka, 10.0, 2.0) for d in ranks])

    by_servant: dict[int, list[int]] = {}
    for t, s in zip(ids.tolist(), srv.tolist()):
        by_servant.setdefault(s, []).append(t)
    batch = []
    for s in sorted(by_servant)[:2000]:
        loc = ranks[0].servant_location(s)
        batch.append((loc, [RunningTask(k, t, loc, f"{t:064x}") for k, t in enumerate(by_servant[s][:50])]))
    out["notify_items"], out["notify_tasks"] = len(batch), sum(len(x[1]) for x in batch)
    # the heartbeat items as C structs, built once: the time is the library call's, not the marshalling's
    items = (_abi.yd_heartbeat_item * len(batch))()
    keep = []
    for i, (loc, tasks) in enumerate(batch):
        arr = (_abi.yd_running_task * max(len(tasks), 1))()
        for k, t in enumerate(tasks):
            enc = (t.servant_location.encode(), t.task_digest.encode())
            keep.append(enc)
            arr[k] = _abi.yd_running_task(t.servant_task_id, t.task_grant_id, *enc)
        lb = loc.encode()
        keep.append((arr, lb))
        items[i] = _abi.yd_heartbeat_item(lb, arr, len(tasks))
    total = out["notify_tasks"]
    unknown = [(C.c_uint64 * total)() for _ in ranks]
    counts = [(C.c_size_t * len(batch))() for _ in ranks]
    out["notify_ms"] = median_slowest(
        [lambda r=r: lib.yd_shard_notify_servants_running_tasks(ranks[r]._h, items, len(batch), unknown[r], counts[r])
         for r in range(W)])
    entries = par([lambda d=d: lib.yd_shard_get_running_tasks(d._h, None, 0) for d in ranks])[0]
    out["running_entries"] = int(entries)
    bufs = [(_abi.yd_running_task * entries)() for _ in ranks]
    out["get_running_tasks_ms"] = median_slowest(
        [lambda r=r: lib.yd_shard_get_running_tasks(ranks[r]._h, bufs[r], entries) for r in range(W)])
    out["running_index_refresh_ms"] = median_slowest([lambda d=d: lib.yd_shard_running_index_refresh(d._h) for d in ranks])
    close(lib, ranks)

    # cfg2-mod's queue as a window of one-decision RPCs, each repetition on a fresh group
    state = {}

    def fresh():
        if "ranks" in state:
            close(lib, state["ranks"])
        rk = group(lib, W, w)
        q = w.build_requests(rk[0])
        rpcs = np.zeros(len(q), dtype=RPC_WAIT_DTYPE)
        rpcs["env_id"], rpcs["min_version"], rpcs["requestor_ip"] = q["env_id"], q["min_version"], q["requestor_ip"]
        rpcs["immediate_reqs"], rpcs["next_keep_alive_ns"] = 1, 10_000_000_000
        state["ranks"], state["rpcs"] = rk, rpcs
    fresh()
    out["rpc_window_rpcs"] = len(state["rpcs"])
    out["rpc_window_ms"] = median_slowest(
        [lambda r=r: state["ranks"][r]._rpcs_with(lib.yd_shard_wait_for_starting_task_rpcs, state["rpcs"], 1.0)
         for r in range(W)], before=fresh)
    close(lib, state["ranks"])

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out["gpu"] = gpu[0] if gpu else "unknown"
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
