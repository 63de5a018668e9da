"""bench.py's N > 1 arm: ONE queue range-sharded over the ranks (include/ydshard.h), strong scaling.

The headline record is BASELINE configs[1] (100 k x 2 k) split over N GPUs -- the same problem as the N = 1
line, so the per-N values are one curve; at that size the four NCCL exchanges cost more than the split saves
(north_star: "only at the 10k+-task scale where it helps"), which the numbers show as they are.  `cfg5_strong`
is BASELINE configs[4] (10 M x 8 k, the configuration the sharding is for) on the same N GPUs.

  value  decisions/s of the whole queue; every rank's range is resident in ITS HBM (yd_stage_requests,
         untimed); time = CUDA events on each rank's solve stream from its first kernel to its grants being
         ready (the four exchanges and the waiting for the slowest rank inside), MAX over ranks.
  e2e    the collective call with pinned HOST buffers: each rank uploads its range and downloads its grants.
"""
from __future__ import annotations

import json
import time

import numpy as np


def measure(name, rank, world, local, steps, warmup, flush, bench):
    import torch
    import torch.distributed as dist

    from yadcc_b200 import STATUS_GRANTED, TaskDispatcher
    from yadcc_b200.sharded import RangeShardedDispatcher

    dev = torch.device("cuda", local)
    w = bench.build_workload(name)
    d = TaskDispatcher(device=local)
    w.register(d, now=0.0, expires_in=3600.0)
    full = w.build_requests(d)
    n = len(full)
    lo, hi = n * rank // world, n * (rank + 1) // world
    reqs = d.alloc_requests(hi - lo)
    reqs[...] = full[lo:hi]
    del full
    out = d.alloc_grants(hi - lo)
    sd = RangeShardedDispatcher(d, rank, world, device=dev)
    dev_ms, e2e_ms = [], []
    prev = None
    stats = None
    granted_total = 0
    for it in range(warmup + steps):
        now = 2.0 + it
        for staged in (False, True):
            if prev is not None:
                sd.free_tasks(prev)
            d.on_expiration_timer(now=now)
            flush.fill_(it & 0xFF)
            if staged:
                d.stage_requests(reqs)
            torch.cuda.synchronize(dev)
            dist.barrier()
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            g = sd.wait_for_starting_new_tasks(len(reqs) if staged else reqs, now, out=out)
            t1 = time.perf_counter()
            assert g is not None, "the sharded solve handed the batch back"
            prev = g["task_id"][g["status"] == STATUS_GRANTED].copy()
            stats = sd.last_stats()
            granted_total = stats["granted_total"]
            if it >= warmup:
                (dev_ms if staged else e2e_ms).append(stats["total_ms"] if staged else 1e3 * (t1 - t0))
    tot = torch.tensor([sum(dev_ms), sum(e2e_ms)] + stats["exchange_ms"], dtype=torch.float64, device=dev)
    dist.all_reduce(tot, op=dist.ReduceOp.MAX)
    tot = tot.tolist()
    sd.free_tasks(prev)
    sd.close()
    d.close()
    K = len(dev_ms)
    rec = {
        "workload": bench.workload_string(name, w), "decisions_per_step": n, "granted_per_step": int(granted_total),
        "value": n * K / (tot[0] / 1e3), "unit": bench.UNIT, "ms_per_step": tot[0] / K,
        "e2e": {"value": n * K / (tot[1] / 1e3), "unit": bench.UNIT, "ms_per_step": tot[1] / K,
                "h2d_bytes_per_step": int(24 * n), "d2h_bytes_per_step": int(16 * n)},
        "collectives": {"library": "NCCL (dlopen'd by libydsched.so), issued on the solve stream",
                        "per_solve": ["all-gather class tables", "all-gather per-class request counts",
                                      "all-reduce reachable request records (disjoint writes)",
                                      "all-reduce per-servant claimed-slot counts u32[S] (+ grant counts, flags)"],
                        "exchange_ms_last_step_max_over_ranks": [round(x, 4) for x in tot[2:6]],
                        "exchange_bytes": stats["exchange_bytes"]},
        "gpu_launches_per_step": stats["kernel_launches"], "merge_rounds": stats["merge_rounds"],
    }
    return rec


def run_sharded(args, rank, world, local):
    import torch
    import torch.distributed as dist

    import bench

    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sampler = bench.ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    main = measure(args.workload, rank, world, local, args.steps, args.warmup, flush, bench)
    if sampler:
        sampler.stop_flag.set()
        sampler.join(timeout=2)
    big = None
    if args.sub != "none" and args.workload == "cfg2-mod":
        big = measure("cfg5", rank, world, local, max(3, args.sub_steps), 3, flush, bench)
    if rank == 0:
        line = {
            "metric": bench.METRIC, "value": main["value"], "unit": bench.UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": main["ms_per_step"], "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "u32", "data": "synthetic",
            "config": {"workload": main["workload"], "decisions_per_step": main["decisions_per_step"],
                       "granted_per_step": main["granted_per_step"],
                       "parallelism": f"one FIFO queue range-sharded over {world} GPUs, servant table replicated",
                       "l2": "flushed between steps (256 MiB write)", "solver": "slot-stream",
                       "between_steps_untimed": "collective FreeTask of the previous grants + OnExpirationTimer tick"},
            "e2e": main["e2e"], "gpu_launches": int(main["gpu_launches_per_step"]) * 2 * args.steps,
            "collectives": main["collectives"],
            "cfg5_strong": big,
            "clocks": sampler.summary(),
            "parity": "tests/multi_gpu_check.py (every decision against one scheduler fed the whole queue; cfg5-1m against "
                      "the reference's digest)",
        }
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()
