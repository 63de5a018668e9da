#!/usr/bin/env python
"""State handover time of the range-sharded scheduler (yd_shard_export_state / yd_shard_import_state, include/ydshard.h)
at W ranks: cfg2-mod (100 k requests over 2 k servants, every request granted) and "1m" (4 k servants with 256 free
slots each, one 1 M-request queue that fills them all).

The ranks are threads of one process on ONE GPU over the test-only NCCL stand-in (tests/fake_nccl, as in
tests/shard_state_check.py), so the host times below include the stand-in's host copies and say nothing about NVLink
exchange time.  Per workload: one sharded solve, then `--steps` collective exports (the size query and the write are
timed as separate calls) and imports into fresh groups; host wall-clock per call (every call ends in a device
synchronise), median and max over the ranks' slowest.  The device time of k_state_merge and k_state_scatter comes from
tools/dev/state_kernels.cu (built with nvcc into a temporary directory): CUDA events, median of `--steps` launches at the
same lease count.  One JSON line per workload, with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.argv, _argv = sys.argv[:1], sys.argv
import shard_state_check as SC  # noqa: E402  (loads the NCCL stand-in first; this process must not import torch)
sys.argv = _argv

from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402


def kernel_times(n: int, world: int, servants: int, reps: int) -> dict:
    src = ROOT / "tools" / "dev" / "state_kernels.cu"
    with tempfile.TemporaryDirectory() as tmp:
        so = Path(tmp) / "state_kernels.so"
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-Xcompiler", "-fPIC", "-shared", f"-I{ROOT / 'include'}", f"-I{ROOT / 'yadcc_b200' / 'csrc'}",
                               "-o", str(so), str(src)])
        lib = C.CDLL(str(so))
        merge, scatter = (C.c_float * reps)(), (C.c_float * reps)()
        rc = lib.time_state_kernels(C.c_ulonglong(n), C.c_uint(world), C.c_uint(servants), C.c_int(reps), merge, scatter)
        assert rc == 0, f"time_state_kernels: {rc}"
    return {"merge_ms_median": round(float(np.median(list(merge))), 4),
            "scatter_ms_median": round(float(np.median(list(scatter))), 4)}


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def run(name: str, world: int, steps: int) -> dict:
    w = S.config2(variant="mod") if name == "cfg2-mod" else SC.million_workload()
    lib = _abi.load_library()
    ranks = SC.new_group(lib, world)
    for d in ranks:
        for sv in w.servants:
            d.keep_servant_alive(sv, 3600.0, now=0.0)
    full = [w.build_requests(d) for d in ranks][0]  # (every rank interns the same strings: replicated tables)
    cut = [len(full) * r // world for r in range(world + 1)]
    parts = [np.ascontiguousarray(full[cut[r]:cut[r + 1]]) for r in range(world)]
    outs = [np.zeros(max(len(p), 1), dtype=_abi.GRANT_DTYPE) for p in parts]
    SC.T.par([lambda r=r: lib.yd_shard_wait_for_starting_new_tasks(ranks[r]._h, SC.T.ns(1.0), parts[r].ctypes.data,
                                                                    len(parts[r]), outs[r].ctypes.data) for r in range(world)])
    leases = sum(d.num_tasks() for d in ranks)
    t = SC.T.ns(2.0)
    size_s, write_s, import_s = [], [], []
    blob = None
    for _ in range(steps):
        sizes, dt = timed(lambda: SC.T.par([lambda d=d: lib.yd_shard_export_state(d._h, t, None, 0) for d in ranks]))
        size_s.append(dt)
        bufs = [C.create_string_buffer(n) for n in sizes]
        _, dt = timed(lambda: SC.T.par([lambda d=d, b=b, n=n: lib.yd_shard_export_state(d._h, t, b, n)
                                        for d, b, n in zip(ranks, bufs, sizes)]))
        write_s.append(dt)
        blob = bufs[0].raw
        fresh = SC.new_group(lib, world)
        rcs, dt = timed(lambda: SC.shard_import(lib, fresh, [blob] * world, 2.0))
        assert rcs == [0] * world, rcs
        import_s.append(dt)
        SC.close_group(lib, fresh)
    SC.close_group(lib, ranks)
    ms = lambda v: {"median": round(1e3 * float(np.median(v)), 2), "max": round(1e3 * max(v), 2)}  # noqa: E731
    line = {"workload": name, "world": world, "leases": leases, "export_bytes": len(blob),
            "host_ms": {"export_size_query": ms(size_s), "export_write": ms(write_s), "import": ms(import_s)},
            "device": kernel_times(leases, world, len(w.servants), steps),
            "exchange": "test-only NCCL stand-in, ranks as threads on one GPU: NVLink exchange time not measured"}
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--workloads", default="cfg2-mod,1m")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    for name in a.workloads.split(","):
        line = run(name, a.world, a.steps)
        line["gpu"] = gpu[0] if gpu else None
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
