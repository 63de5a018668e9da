#!/usr/bin/env python
"""Export and import time of a scheduler handle's state (include/ydstate.h) at BASELINE configs[1] (cfg2-mod: 100 k
requests over 2 k servants) and configs[2] (cfg3: 1 M requests over 4 k servants) scale, and with one million live
leases ("1m-leases": 4 k servants with 256 free slots each, one 1 M-request queue that fills them all).

Per workload: register the servants, grant one full queue (every grant stays live), then `--steps` exports and imports
of that state.  Reports host wall-clock per call (the calls end in a device synchronise) and the device time of the
state kernels and copies from torch.profiler, with the card's name and power limit.  One JSON line per workload."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from yadcc_b200 import TaskDispatcher  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200.dispatcher import Servant  # noqa: E402
from bench import build_workload  # noqa: E402


def setup(name: str):
    """A handle holding the leases of one granted queue; returns (handle, servants, live leases)."""
    d = TaskDispatcher()
    if name == "1m-leases":
        servants = [Servant(f"{S.servant_ip(k)}:8335", environments=["e" * 64], num_processors=256, max_tasks=256)
                    for k in range(4000)]
        d.keep_servants_alive(servants, 3600.0, now=0.0)
        src = d.make_requests(1_000_000, "e" * 64, "172.16.0.1", expires_in=60)
    else:
        w = build_workload(name, 0)
        w.register(d, now=0.0, expires_in=3600.0)
        servants, src = w.servants, w.build_requests(d)
    reqs = d.alloc_requests(len(src))
    reqs[...] = src
    g = d.wait_for_starting_new_tasks(reqs, now=1.0)
    return d, len(servants), int((g["status"] == 2).sum())


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def device_ms(fn) -> dict:
    """Device time of the calls in fn(), by kind, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"kernels_ms": 0.0, "copies_ms": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        dt = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        if "emcpy" in e.name:
            out["copies_ms"] += dt
        elif "k_" in e.name:
            out["kernels_ms"] += dt
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("workloads", nargs="*", default=["cfg2-mod", "cfg3", "1m-leases"])
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    info = card()
    for name in args.workloads:
        d, n_servants, leases = setup(name)
        blob = d.export_state(now=2.0)  # warm-up (first use of the stream-ordered pool)
        t_exp, t_imp = [], []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            blob = d.export_state(now=2.0)
            t1 = time.perf_counter()
            e = TaskDispatcher()
            t2 = time.perf_counter()
            e.import_state(blob, now=2.0)
            t3 = time.perf_counter()
            t_exp.append(t1 - t0)
            t_imp.append(t3 - t2)
            e.close()
        holder = {}

        def one_export():
            holder["blob"] = d.export_state(now=2.0)

        dev_exp = device_ms(one_export)
        e = TaskDispatcher()
        dev_imp = device_ms(lambda: e.import_state(holder["blob"], now=2.0))
        ok = e.export_state(now=2.0) == blob
        e.close()
        d.close()
        print(json.dumps({"workload": name, "servants": n_servants, "live_leases": leases, "export_bytes": len(blob),
                          "export_ms_median": 1e3 * float(np.median(t_exp)), "import_ms_median": 1e3 * float(np.median(t_imp)),
                          "export_device": dev_exp, "import_device": dev_imp, "round_trip_identical": ok,
                          "steps": args.steps, **info}), flush=True)


if __name__ == "__main__":
    main()
