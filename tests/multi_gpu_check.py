#!/usr/bin/env python
"""Parity of the range-sharded scheduler (include/ydshard.h) against ONE scheduler fed the whole queue.

Run under torchrun on a box with >= 2 GPUs (tests/test_multi_gpu.py does, when it sees them):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multi_gpu_check.py [--quick]

Every rank builds the same workload, registers the same servants (replicated table), takes the
g-th contiguous range of the FIFO queue and joins the collective solve.  Rank 0 also solves the
whole queue on a second, ordinary handle and compares statuses, servants and task ids of every
request, the per-servant bookkeeping, and -- for cfg5-1m -- the digest the REFERENCE produced
(tests/golden/digests.json).  Two rounds with a collective FreeTask of half the grants in between.
Exit code 0 iff everything is identical.
"""
import argparse
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from yadcc_b200 import STATUS_GRANTED, TaskDispatcher  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT_DTYPE  # noqa: E402
from yadcc_b200.sharded import RangeShardedDispatcher  # noqa: E402


def ranges(n, world, skew):
    """Contiguous split; `skew` moves the cut points around (one variant leaves a rank empty)."""
    if skew == "even":
        cuts = [n * g // world for g in range(world + 1)]
    elif skew == "empty-last":
        cuts = [n * g // (world - 1) if g < world else n for g in range(world)] + [n]
    else:  # uneven
        w = np.arange(1, world + 1, dtype=np.float64) ** 1.5
        cuts = [0] + [int(x) for x in np.round(np.cumsum(w) / w.sum() * n)]
        cuts[-1] = n
    return cuts


def gather_grants(local: np.ndarray, counts, rank, world, dev):
    """All ranks' grant arrays on rank 0 (padded all_gather of the raw bytes)."""
    m = max(counts) * GRANT_DTYPE.itemsize
    buf = torch.zeros(max(m, 16), dtype=torch.uint8, device=dev)
    raw = np.frombuffer(local.tobytes(), dtype=np.uint8)
    buf[: len(raw)] = torch.from_numpy(raw.copy()).to(dev)
    outs = [torch.zeros_like(buf) for _ in range(world)]
    dist.all_gather(outs, buf)
    parts = [np.frombuffer(o.cpu().numpy().tobytes()[: c * GRANT_DTYPE.itemsize], dtype=GRANT_DTYPE) for o, c in zip(outs, counts)]
    return np.concatenate(parts) if parts else np.zeros(0, GRANT_DTYPE)


def check(name, w, skew, rank, world, dev, golden=None):
    d = TaskDispatcher(device=dev.index)
    w.register(d, now=0.0, expires_in=3600.0)
    full = w.build_requests(d)
    n = len(full)
    cuts = ranges(n, world, skew)
    mine = np.ascontiguousarray(full[cuts[rank]:cuts[rank + 1]])
    counts = [cuts[g + 1] - cuts[g] for g in range(world)]
    sd = RangeShardedDispatcher(d, rank, world, device=dev)
    single = None
    if rank == 0:
        single = TaskDispatcher(device=dev.index)
        w.register(single, now=0.0, expires_in=3600.0)
        full_single = w.build_requests(single)  # (digest / IP ids are per handle)
    ok_all = True
    for rnd in range(2):
        now = 0.001 + rnd
        g_local = sd.wait_for_starting_new_tasks(mine, now)
        g_all = gather_grants(g_local, counts, rank, world, dev)
        st = d.servant_state()
        alive = torch.tensor([d.num_tasks()], dtype=torch.int64, device=dev)
        dist.all_reduce(alive)
        stats = sd.last_stats()
        if rank == 0:
            g_one = single.wait_for_starting_new_tasks(full_single, now)
            st1 = single.servant_state()
            same = (bool((g_all["status"] == g_one["status"]).all()) and bool((g_all["servant_index"] == g_one["servant_index"]).all())
                    and bool((g_all["task_id"] == g_one["task_id"]).all()))
            same_state = bool((st["running_tasks"] == st1["running_tasks"]).all()) and bool(
                (st["ever_assigned_tasks"] == st1["ever_assigned_tasks"]).all())
            same_ids = d.next_task_id() == single.next_task_id() and int(alive.item()) == single.num_tasks()
            line = {"workload": name, "split": skew, "round": rnd, "world": world, "requests": n,
                    "granted": int((g_one["status"] == STATUS_GRANTED).sum()), "grants_equal": same, "state_equal": same_state,
                    "ids_equal": same_ids, "exchange_ms": [round(x, 4) for x in stats["exchange_ms"]],
                    "exchange_bytes": stats["exchange_bytes"], "total_ms": round(stats["total_ms"], 4)}
            if not same:
                bad = {k: int((g_all[k] != g_one[k]).sum()) for k in ("status", "servant_index", "task_id")}
                first = int(np.nonzero((g_all["status"] != g_one["status"]) | (g_all["servant_index"] != g_one["servant_index"])
                                       | (g_all["task_id"] != g_one["task_id"]))[0][0])
                line["mismatches"] = bad
                line["first"] = {"index": first, "cuts": cuts, "sharded": [int(x) for x in g_all[first]], "single": [int(x) for x in g_one[first]]}
            if golden is not None and rnd == 0:
                trace = [g_all, np.stack([st["running_tasks"], st["ever_assigned_tasks"], st["capacity_available"]], axis=1),
                         np.asarray([d.next_task_id(), int(alive.item()), d.num_servants()], dtype=np.uint64)]
                line["reference_digest_equal"] = S.trace_digest(trace) == golden["sha256"]
                same = same and line["reference_digest_equal"]
            print(json.dumps(line), flush=True)
            ok_all = ok_all and same and same_state and same_ids
        # replicas must agree on running_tasks
        rt = torch.from_numpy(st["running_tasks"].astype(np.int64)).to(dev)
        lo, hi = rt.clone(), rt.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        if not bool((lo == hi).all()):
            ok_all = False
            if rank == 0:
                print(json.dumps({"workload": name, "error": "running_tasks differ between ranks"}), flush=True)
        # collective FreeTask: every rank releases a seeded half of ITS grants; the single scheduler the union
        okm = g_local["status"] == STATUS_GRANTED
        ids = g_local["task_id"][okm]
        pick = ids[np.random.default_rng(100 + rnd).random(len(ids)) < 0.5] if rank % 2 == 0 else ids[: len(ids) // 3]
        sd.free_tasks(pick)
        freed = gather_ids(pick, rank, world, dev)
        d.on_expiration_timer(now=now + 0.5)
        if rank == 0:
            single.free_tasks(freed)
            single.on_expiration_timer(now=now + 0.5)
    flag = torch.tensor([1 if ok_all else 0], dtype=torch.int64, device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    sd.close()
    d.close()
    if single:
        single.close()
    return bool(flag.item())


def gather_ids(ids: np.ndarray, rank, world, dev):
    cnt = torch.tensor([len(ids)], dtype=torch.int64, device=dev)
    cnts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(cnts, cnt)
    m = max(int(c.item()) for c in cnts)
    buf = torch.zeros(max(m, 1), dtype=torch.int64, device=dev)
    buf[: len(ids)] = torch.from_numpy(ids.astype(np.int64)).to(dev)
    outs = [torch.zeros_like(buf) for _ in range(world)]
    dist.all_gather(outs, buf)
    return np.concatenate([o.cpu().numpy()[: int(c.item())] for o, c in zip(outs, cnts)]).astype(np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    golden = json.loads((ROOT / "tests" / "golden" / "digests.json").read_text())["streams"]
    cases = [
        ("cfg2-mod-small", S.config2(5000, 200, 8, variant="mod"), "even", None),
        ("cfg2-random-small", S.config2(5000, 200, 8, variant="random"), "uneven", None),
        ("cfg-self-small", S.config_self(6000, 150), "even", None),
        ("cfg3-20k", S.config3(20000, 300, 8), "uneven", None),
        ("cfg2-mod", S.config2(variant="mod"), "even", None),
        ("cfg2-random", S.config2(variant="random"), "uneven", None),
        ("cfg-self", S.config_self(), "even", None),
    ]
    if world > 2:
        cases.append(("cfg2-random-small", S.config2(5000, 200, 8, variant="random"), "empty-last", None))
    if not args.quick:
        cases += [("cfg3-1m", S.config3(1_000_000, 4000, 8), "even", None),
                  ("cfg5-1m", S.config5(1_000_000, 8000), "even", golden.get("cfg5-1m"))]
    ok = True
    for name, w, skew, gold in cases:
        ok = check(name, w, skew, rank, world, dev, gold) and ok
    if rank == 0:
        print(json.dumps({"multi_gpu_parity": ok, "world": world}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
