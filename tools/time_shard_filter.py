#!/usr/bin/env python
"""Time of the range-sharded group's pre-filtered solve from task descriptors
(yd_shard_derive_filter_and_wait_for_starting_new_tasks, include/ydshard.h) at W = 1, 2, 4 ranks, against the
single-handle call (yd_derive_filter_and_wait_for_starting_new_tasks) on the whole queue.

The ranks are threads of one process on ONE GPU over the test-only NCCL stand-in (tests/fake_nccl), so this shows each
rank's stage time shrinking with its range; it does not show a multi-GPU speed-up (the ranks share one device), and the
exchange times include the stand-in's host copies.  Queues: the configs[3] descriptor queue
(streams.config3_task_sources) at 100 k and 1 M requests over cfg2-mod's 2 000 servants; both stages, an empty bloom
filter and an empty in-flight index, so every request is offered.  Per rank and call: the device time of its stages
(yd_last_solve_stats().prep_ms), the sharded solve's device time (yd_shard_last_stats().total_ms) and the host
wall-clock around the collective call; the grants are freed after every call, so each repetition decides the same
queue on the same state.  Medians of `--reps` after one warm-up call.  One JSON line with the card's name and power
limit.
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
from yadcc_b200.dispatcher import TaskDispatcher, TaskSources  # noqa: E402

STAGES = _abi.STAGE_CACHE | _abi.STAGE_DEDUPE


def par(fns):
    import threading

    out = [None] * len(fns)
    ts = [threading.Thread(target=lambda i=i, f=f: out.__setitem__(i, f())) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def med(xs):
    return round(float(np.median(xs)), 3)


def handle(lib, w):
    d = TaskDispatcher(lib)
    w.register(d, now=0.0, expires_in=3600.0)
    d.bloom_reset(27584639, 10)
    return d


def single(lib, w, q, src, reps):
    d = handle(lib, w)
    prep, host = [], []
    for k in range(reps + 1):
        t0 = time.perf_counter()
        _, _, g = d.derive_filter_and_wait_for_starting_new_tasks(q, src, STAGES, 1.0 + k)
        t = (time.perf_counter() - t0) * 1e3
        if k:
            prep.append(d.last_solve_stats()["prep_ms"])
            host.append(t)
        d.free_tasks(g["task_id"][g["status"] == _abi.STATUS_GRANTED].copy())
    d.close()
    return {"prep_ms": med(prep), "host_ms": med(host)}


def grouped(lib, w, q, src, world, reps):
    ranks = [handle(lib, w) for _ in range(world)]
    uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
    assert lib.yd_shard_unique_id(uid) == 0
    assert par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, world, uid) for r in range(world)]) == [0] * world
    n = len(q)
    cuts = [n * g // world for g in range(world + 1)]
    parts = [np.ascontiguousarray(q[cuts[r]:cuts[r + 1]]) for r in range(world)]
    srcs = [TaskSources(src.args, src.args_offsets, np.ascontiguousarray(src.args_index[cuts[r]:cuts[r + 1]]),
                        np.ascontiguousarray(src.source_digests[cuts[r]:cuts[r + 1]])) for r in range(world)]
    fn = lib.yd_shard_derive_filter_and_wait_for_starting_new_tasks
    per = [{"prep_ms": [], "shard_total_ms": [], "host_ms": []} for _ in range(world)]
    st = _abi.yd_shard_stats()
    for k in range(reps + 1):
        def call(r):
            t0 = time.perf_counter()
            out = ranks[r]._derive_filter_with(fn, parts[r], srcs[r], STAGES, 1.0 + k, None, None, True)
            return out, (time.perf_counter() - t0) * 1e3
        res = par([lambda r=r: call(r) for r in range(world)])
        for r in range(world):
            if k:
                assert lib.yd_shard_last_stats(ranks[r]._h, C.byref(st)) == 1
                per[r]["prep_ms"].append(ranks[r].last_solve_stats()["prep_ms"])
                per[r]["shard_total_ms"].append(st.total_ms)
                per[r]["host_ms"].append(res[r][1])
        ids = [np.ascontiguousarray(g["task_id"][g["status"] == _abi.STATUS_GRANTED]) for (_, _, g), _ in res]
        assert par([lambda r=r: lib.yd_shard_free_tasks(ranks[r]._h, ids[r].ctypes.data if len(ids[r]) else None,
                                                        len(ids[r])) for r in range(world)]) == [0] * world
    for d in ranks:
        lib.yd_shard_finalize(d._h)
        d.close()
    return [{k: med(v) for k, v in p.items()} for p in per]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--worlds", default="1,2,4")
    a = ap.parse_args()
    lib = _abi.load_library()
    out = {"nccl": "fake_nccl (threads on one GPU)", "reps": a.reps, "stages": "cache+dedupe", "queues": []}
    for n in [int(x) for x in a.sizes.split(",")]:
        w = S.config2(n, 2000, 8, seed=42, variant="mod")
        src = S.config3_task_sources(n)
        probe = TaskDispatcher(lib)
        w.register(probe, now=0.0, expires_in=3600.0)
        q = np.ascontiguousarray(w.build_requests(probe))
        probe.close()
        row = {"requests": n, "single": single(lib, w, q, src, a.reps), "groups": {}}
        for world in [int(x) for x in a.worlds.split(",")]:
            row["groups"][str(world)] = grouped(lib, w, q, src, world, a.reps)
        out["queues"].append(row)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out["gpu"] = gpu[0] if gpu else "unknown"
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
