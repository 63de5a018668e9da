#!/usr/bin/env python
"""Host wall-clock of a window of WaitForStartingTask RPCs, packed (yd_wait_for_starting_task_rpcs_packed: the window
expanded, decided and reported on the device, 32 bytes per RPC up, 16 per RPC and 8 per grant down) against the unpacked
call (yd_wait_for_starting_task_rpcs: expansion and report on the host, 24 bytes per decision up, 16 down).

Cluster: cfg2-mod's 2000 servants (8 digests, 64 tasks each).  Windows:
  rpc10, rpc1k, rpc100k   10, 1 000 and 100 000 RPCs of one immediate request each (cfg2-mod's queue as RPCs)
  rpc1k_pre8              1 000 RPCs of 1 immediate + 8 prefetch requests
  greedy100               100 RPCs asking for 0xFFFFFFFF immediate and 0xFFFFFFFF prefetch requests
The two forms run on twin handles fed the same events, alternated in one process; after every call its grants are freed
and the clock ticks, so every repetition decides the same window on the same state.  Every call's outputs are compared
(results equal, the packed grants unpacked equal the unpacked grants).  Per call: the host clock around it (the call ends
in a stream synchronise) and its yd_last_solve_stats.  With --world W (W >= 1) the same windows run on two range-sharded
groups of W rank threads each over the test-only NCCL stand-in (tests/fake_nccl, loaded before anything else).  One JSON
line per window with the median and range over --reps calls after --warmup, and the card's name and power limit read in
the same run.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
ap = argparse.ArgumentParser()
ap.add_argument("--windows", default="rpc10,rpc1k,rpc100k,rpc1k_pre8,greedy100")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--reps", type=int, default=11)
ap.add_argument("--world", type=int, default=0, help="0: one handle per form; W: a group of W ranks per form")
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
A = ap.parse_args()
if A.world:
    FAKE = C.CDLL(str(ROOT / "tests" / "fake_nccl" / "libnccl.so.2"), mode=C.RTLD_GLOBAL)

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
from yadcc_b200 import STATUS_GRANTED, _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200.dispatcher import TaskDispatcher, unpack_grants  # noqa: E402


def par(fns):
    out = [None] * len(fns)

    def run(i, f):
        out[i] = f()
    ts = [threading.Thread(target=run, args=(i, f)) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def window(name, d, w):
    """The window `name` as RPC records interned on d."""
    reqs = w.build_requests(d)
    env, ip = reqs["env_id"], reqs["requestor_ip"]

    def rpcs(n, imm, pre):
        r = np.zeros(n, dtype=_abi.RPC_WAIT_DTYPE)
        r["env_id"], r["requestor_ip"] = env[:n], ip[:n]
        r["immediate_reqs"], r["prefetch_reqs"] = imm, pre
        r["next_keep_alive_ns"] = 15_000_000_000
        return r
    return {"rpc10": lambda: rpcs(10, 1, 0), "rpc1k": lambda: rpcs(1000, 1, 0), "rpc100k": lambda: rpcs(100_000, 1, 0),
            "rpc1k_pre8": lambda: rpcs(1000, 1, 8), "greedy100": lambda: rpcs(100, 0xFFFFFFFF, 0xFFFFFFFF)}[name]()


def group(lib, W):
    ranks = [TaskDispatcher(lib) for _ in range(W)]
    uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
    assert lib.yd_shard_unique_id(uid) == 0
    assert par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, W, uid) for r in range(W)]) == [0] * W
    return ranks


def stats(xs):
    return {"median": round(float(np.median(xs)), 4), "min": round(float(min(xs)), 4), "max": round(float(max(xs)), 4)}


def run(name, W):
    lib = _abi.load_library()
    w = S.config2(100_000, 2000, 8, variant="mod")
    P = group(lib, W) if W else [TaskDispatcher(lib)]
    U = group(lib, W) if W else [TaskDispatcher(lib)]
    for d in P + U:
        w.register(d, now=0.0, expires_in=3600.0)
    rp, ru = [window(name, d, w) for d in P], [window(name, d, w) for d in U]
    fp = (lambda d, r, now: d._rpcs_packed_with(lib.yd_shard_wait_for_starting_task_rpcs_packed, r, now)) if W else \
        (lambda d, r, now: d.wait_for_starting_task_rpcs_packed(r, now))
    fu = (lambda d, r, now: d._rpcs_with(lib.yd_shard_wait_for_starting_task_rpcs, r, now)) if W else \
        (lambda d, r, now: d.wait_for_starting_task_rpcs(r, now))
    t = {"packed": [], "unpacked": []}
    dev = {"packed": [], "unpacked": []}
    now = 1.0
    for k in range(A.warmup + A.reps):
        now += 0.01
        t0 = time.perf_counter()
        outp = par([lambda r=r: fp(P[r], rp[r], now) for r in range(len(P))])
        t1 = time.perf_counter()
        sp = P[0].last_solve_stats()
        t2 = time.perf_counter()
        outu = par([lambda r=r: fu(U[r], ru[r], now) for r in range(len(U))])
        t3 = time.perf_counter()
        su = U[0].last_solve_stats()
        res8, g8, ids = outp[0]
        res, g = outu[0]
        for x in outp[1:]:
            assert x[0].tobytes() == res8.tobytes() and x[1].tobytes() == g8.tobytes(), f"ranks differ at call {k}"
        gu = unpack_grants(g8, ids)
        assert res8.tobytes() == res.tobytes() and (gu == g).all(), f"outputs differ at call {k}"
        if k >= A.warmup:
            t["packed"].append((t1 - t0) * 1e3)
            t["unpacked"].append((t3 - t2) * 1e3)
            if not W:
                dev["packed"].append(sp)
                dev["unpacked"].append(su)
        ids_done = np.ascontiguousarray(g["task_id"][g["status"] == STATUS_GRANTED])
        for ds in (P, U):
            if W:  # (rank 0 passes the ids of the collective free)
                par([lambda r=r: lib.yd_shard_free_tasks(ds[r]._h, ids_done.ctypes.data if r == 0 else None,
                                                         len(ids_done) if r == 0 else 0) for r in range(W)])
            else:
                ds[0].free_tasks(ids_done)
            for d in ds:
                d.on_expiration_timer(now=now + 0.005)
    total = int(lib.yd_rpc_expanded_requests(P[0]._h, rp[0].ctypes.data, len(rp[0])))
    out = {"window": name, "world": W, "rpcs": len(rp[0]), "decisions": total, "granted": len(g8), "reps": A.reps}
    for form in ("packed", "unpacked"):
        out[form] = {"host_ms": stats(t[form])}
        if dev[form]:
            s = dev[form][-1]
            out[form].update(device_total_ms=stats([x["total_ms"] for x in dev[form]]), h2d_bytes=s["h2d_bytes"],
                             d2h_bytes=s["d2h_bytes"], kernel_launches=s["kernel_launches"])
    out["host_speedup_median"] = round(float(np.median(t["unpacked"]) / np.median(t["packed"])), 3)
    for d in P + U:
        if W:
            lib.yd_shard_finalize(d._h)
        d.close()
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    for name in A.windows.split(","):
        line = json.dumps({"tool": "time_rpcs_packed", "gpu": gpu[0] if gpu else "unknown",
                           "nccl": "fake_nccl" if A.world else None, **run(name, A.world)})
        print(line, flush=True)
        if A.out:
            with open(A.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
