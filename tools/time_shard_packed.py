#!/usr/bin/env python
"""Host wall-clock of the range-sharded group's collective solve, packed (yd_shard_wait_for_starting_new_tasks_packed:
16-byte requests up, 8-byte grants down) against unpacked (yd_shard_wait_for_starting_new_tasks: 24 up, 16 down), at
W = 1, 2, 4 ranks.

The ranks are threads of one process on ONE GPU over the test-only NCCL stand-in (tests/fake_nccl): they share one
device and one PCIe link, and the exchanges include the stand-in's host copies, so this shows what the narrower records
save per rank, not a multi-GPU number.  Queues: cfg2-mod (100 k x 2 k) and cfg5 (10 M x 8 k), cut into W even ranges,
each rank's range in page-locked arrays (yd_alloc_host).  Per call and rank: the host clock around the collective call;
the two forms alternate in one process, and every call is preceded by a collective free of the previous call's grants
and a tick, so every repetition decides the same queue on the same state.  Reported: the slowest rank's time per call,
median and range over `--reps` calls after `--warmup`, and the H2D / D2H bytes per decision from the record sizes.  One
JSON line with the card's name and power limit.
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
from yadcc_b200.dispatcher import TaskDispatcher, pack_requests  # noqa: E402

WORKLOADS = {"cfg2-mod": lambda: S.config2(variant="mod"), "cfg5": lambda: S.config5()}


def par(fns):
    import threading

    out = [None] * len(fns)
    ts = [threading.Thread(target=lambda i=i, f=f: out.__setitem__(i, f())) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def group(lib, name, world, warmup, reps):
    w = WORKLOADS[name]()
    ranks = [TaskDispatcher(lib) for _ in range(world)]
    for d in ranks:
        w.register(d, now=0.0, expires_in=1e6)
    uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
    assert lib.yd_shard_unique_id(uid) == 0
    assert par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, world, uid) for r in range(world)]) == [0] * world
    req, req16, out, out8 = [], [], [], []
    for r, d in enumerate(ranks):
        full = w.build_requests(d)  # (interns on this handle, in the same order as on the others)
        n = len(full)
        lo, hi = n * r // world, n * (r + 1) // world
        a = d.alloc_requests(hi - lo)
        a[...] = full[lo:hi]
        req.append(a)
        b = d.alloc_requests16(hi - lo)
        pack_requests(a, out=b)
        req16.append(b)
        out.append(d.alloc_grants(hi - lo))
        out8.append(d.alloc_grants8(hi - lo))
        del full
    ids = [np.zeros(1, dtype=_abi.PACKED_IDS_DTYPE) for _ in range(world)]
    n_total = sum(len(a) for a in req)
    times = {"packed": [], "unpacked": []}
    granted = {}
    for k in range(warmup + reps):
        for form in ("packed", "unpacked"):
            now = 1.0 + 2 * k + (form == "unpacked")

            def call(r):
                ranks[r].on_expiration_timer(now=now)
                t0 = time.perf_counter()
                if form == "packed":
                    rc = lib.yd_shard_wait_for_starting_new_tasks_packed(ranks[r]._h, int(now * 1e9), req16[r].ctypes.data,
                                                                         len(req16[r]), out8[r].ctypes.data,
                                                                         ids[r].ctypes.data)
                else:
                    rc = lib.yd_shard_wait_for_starting_new_tasks(ranks[r]._h, int(now * 1e9), req[r].ctypes.data,
                                                                  len(req[r]), out[r].ctypes.data)
                t = (time.perf_counter() - t0) * 1e3
                assert rc == 0, rc
                if form == "packed":
                    so = out8[r]["status_ordinal"][: len(req16[r])]
                    g = so >> 30 == _abi.STATUS_GRANTED
                    tid = ids[r][0]["first_task_id"] + (so[g] & 0x3FFFFFFF).astype(np.uint64) * ids[r][0]["stride"]
                else:
                    g = out[r]["status"][: len(req[r])] == _abi.STATUS_GRANTED
                    tid = out[r]["task_id"][: len(req[r])][g]
                return t, np.ascontiguousarray(tid, dtype=np.uint64)
            res = par([lambda r=r: call(r) for r in range(world)])
            if k >= warmup:
                times[form].append(max(t for t, _ in res))
            granted[form] = int(sum(len(x) for _, x in res))
            tids = [x for _, x in res]
            assert par([lambda r=r: lib.yd_shard_free_tasks(ranks[r]._h, tids[r].ctypes.data if len(tids[r]) else None,
                                                            len(tids[r])) for r in range(world)]) == [0] * world
    assert granted["packed"] == granted["unpacked"], granted
    for d in ranks:
        lib.yd_shard_finalize(d._h)
        d.close()
    row = {"world": world, "requests": n_total, "granted": granted["packed"]}
    for form, xs in times.items():
        row[form] = {"median_ms": round(float(np.median(xs)), 3), "min_ms": round(min(xs), 3),
                     "max_ms": round(max(xs), 3), "calls": len(xs)}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2-mod,cfg5")
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    lib = _abi.load_library()
    rq, rq16, g, g8 = (x.itemsize for x in (_abi.REQ_DTYPE, _abi.REQ16_DTYPE, _abi.GRANT_DTYPE, _abi.GRANT8_DTYPE))
    out = {"nccl": "fake_nccl (threads on one GPU)", "time": "slowest rank's host wall-clock per collective call",
           "bytes_per_decision": {"packed": {"h2d": rq16, "d2h": g8, "total": rq16 + g8},
                                  "unpacked": {"h2d": rq, "d2h": g, "total": rq + g}},
           "rows": []}
    for name in a.workloads.split(","):
        for world in [int(x) for x in a.worlds.split(",")]:
            row = group(lib, name, world, a.warmup, a.reps)
            row["workload"] = name
            out["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out["gpu"] = gpu[0] if gpu else "unknown"
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
