#!/usr/bin/env python
"""End-to-end time of the pre-filtered solve (BASELINE configs[3]), packed (yd_filter_and_wait_for_starting_new_tasks_packed:
16-byte requests and two 32-byte binary digests up, 8-byte grants down) against the key-based call
(yd_filter_and_wait_for_starting_new_tasks: 24-byte requests, the 81-byte cache key and the 64-byte task digest up,
16-byte grants down), on one handle each.

Queue: the cfg4 set-up of tests/test_filter_packed.py (cfg2-mod's 2000 servants, 6124 TUs with 30 % of their cache keys
in the bloom filter, an in-flight index over 1500 running tasks) at 100 k and 1 M requests, every input in page-locked
host arrays (yd_alloc_host), both stages on, hits not requested.  The two handles get the same events; the forms
alternate in one process, and after every call its grants are freed and the clock ticks, so every repetition decides
the same queue on the same state.  Per call: the host clock around it (the call ends in a stream synchronise), and the
device times of the call's own events (yd_last_solve_stats: prep_ms = the filter stages and the compaction, total_ms =
the solve).  The two calls' outputs are compared on every timed call.  One JSON line per size with the median and range
over --reps calls after --warmup, and the card's name and power limit read in the same run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from test_filter_packed import cfg4_setup, hexkeys  # noqa: E402
from yadcc_b200 import STATUS_GRANTED, _abi  # noqa: E402
from yadcc_b200.dispatcher import TaskDispatcher, unpack_grants  # noqa: E402


def pinned(d, a):
    out = d._alloc(a.size, np.dtype(a.dtype)).reshape(a.shape)
    out[...] = a
    return out


def unpacked_reqs(r16):
    r = np.zeros(len(r16), dtype=_abi.REQ_DTYPE)
    r["env_id"], r["min_version"], r["requestor_ip"] = r16["env_id"], r16["min_version"], r16["requestor_ip"]
    r["flags"] = np.where(r16["lease"] & _abi.LEASE_PREFETCH, _abi.REQ_FLAG_PREFETCH, 0)
    r["expires_in_ns"] = (r16["lease"] & 0x7FFFFFFF).astype(np.int64) * 1_000_000
    return r


def stats(xs):
    return {"median": round(float(np.median(xs)), 4), "min": round(float(min(xs)), 4), "max": round(float(max(xs)), 4)}


def run(n, warmup, reps):
    dp, du = TaskDispatcher(), TaskDispatcher()
    r16, cd, td = cfg4_setup(dp, n)
    r16b, _, _ = cfg4_setup(du, n)
    assert (r16 == r16b).all()
    # page-locked inputs and outputs of both forms
    P = {"r16": pinned(dp, r16), "cd": pinned(dp, cd), "td": pinned(dp, td), "v": dp._alloc(n, np.dtype(np.uint8)),
         "g8": dp.alloc_grants8(n)}
    km = np.frombuffer("".join(hexkeys(cd, True)).encode(), np.uint8).reshape(n, 81)
    dm = np.frombuffer("".join(hexkeys(td, False)).encode(), np.uint8).reshape(n, 64)
    U = {"r": pinned(du, unpacked_reqs(r16)), "km": pinned(du, km), "dm": pinned(du, dm), "v": du._alloc(n, np.dtype(np.uint8)),
         "g": du.alloc_grants(n)}
    t = {"packed": [], "unpacked": []}
    dev = {"packed": [], "unpacked": []}
    now = 1.0
    for k in range(warmup + reps):
        now += 0.01  # (well inside the servants' heartbeat expiry)
        t0 = time.perf_counter()
        v8, _, g8, ids = dp.filter_and_wait_for_starting_new_tasks_packed(P["r16"], P["cd"], P["td"], now, False,
                                                                           out8=P["g8"], verdict_out=P["v"])
        t1 = time.perf_counter()
        sp = dp.last_solve_stats()
        t2 = time.perf_counter()
        v, _, g = du.filter_and_wait_for_starting_new_tasks(U["r"], U["km"], U["dm"], now, out=U["g"], verdict_out=U["v"],
                                                            want_hits=False)
        t3 = time.perf_counter()
        su = du.last_solve_stats()
        gu = unpack_grants(g8, ids)
        assert (v8 == v).all() and (gu == g).all(), f"outputs differ at call {k}"
        if k >= warmup:
            t["packed"].append((t1 - t0) * 1e3)
            t["unpacked"].append((t3 - t2) * 1e3)
            dev["packed"].append((sp["prep_ms"], sp["total_ms"], sp["h2d_bytes"], sp["d2h_bytes"]))
            dev["unpacked"].append((su["prep_ms"], su["total_ms"], su["h2d_bytes"], su["d2h_bytes"]))
        for d, gr in ((dp, gu), (du, g)):
            d.free_tasks(np.ascontiguousarray(gr["task_id"][gr["status"] == STATUS_GRANTED]))
            d.on_expiration_timer(now=now + 0.005)
    offered = int((v == _abi.FILTER_OFFERED).sum())
    assert (g["status"] == STATUS_GRANTED).any()
    out = {"n": n, "offered": offered, "granted": int((g["status"] == STATUS_GRANTED).sum()), "reps": reps}
    for form in ("packed", "unpacked"):
        out[form] = {"host_ms": stats(t[form]), "filter_device_ms": stats([x[0] for x in dev[form]]),
                     "solve_device_ms": stats([x[1] for x in dev[form]]), "h2d_bytes": dev[form][-1][2],
                     "d2h_bytes": dev[form][-1][3], "decisions_per_s_host": round(n / (np.median(t[form]) / 1e3))}
    out["host_speedup_median"] = round(float(np.median(t["unpacked"]) / np.median(t["packed"])), 3)
    dp.close()
    du.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert a.reps >= 7
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    for n in (int(x) for x in a.sizes.split(",")):
        line = json.dumps({"tool": "time_filter_packed", "gpu": gpu[0] if gpu else "unknown", **run(n, a.warmup, a.reps)})
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
