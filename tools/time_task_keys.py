#!/usr/bin/env python
"""Cost of deriving the configs[3] cache keys and task digests from task descriptors (development aid; bench.py is the
contract).  On the 100 k-request configs[3] queue with its descriptors (streams.config3_task_sources) it reports:

  * device time of the derivation kernel alone (torch.profiler, CUDA activities, over many calls after warm-up), and
    the same from the calls' own CUDA events: prep_ms of the descriptor pipeline minus that of the key-based one;
  * end-to-end host time of the descriptor pipeline (yd_derive_filter_and_wait_for_starting_new_tasks) next to the
    key-based one-call pipeline (yd_filter_and_wait_for_starting_new_tasks) on the same queue and state, alternated;
  * host time of deriving the same keys with the CPU reference build (oracle/_ref, one thread);
  * H2D bytes of both pipelines;
with the card's name and power limit read in the same run.  Prints the record as one JSON line (and writes it to --out
if given)."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from yadcc_b200 import STATUS_GRANTED, RunningTask, TaskDispatcher, TaskSources  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from bench import build_workload  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def setup(d: TaskDispatcher, n: int):
    """The configs[3] state of bench.py's Cfg4Stages, built from derived keys: a third of the TUs' cache keys in the
    bloom filter, an earlier wave of 1500 tasks listed by the servants' heartbeats."""
    w = build_workload("cfg4")
    w.register(d, now=0.0, expires_in=3600.0)
    reqs = w.build_requests(d)[:n].copy()
    src = S.config3_task_sources(n)
    keys, digests = d.derive_task_keys(reqs, src)
    d.bloom_reset()
    d.bloom_add(keys[: 6124][np.random.default_rng(4).random(min(n, 6124)) < 0.3])
    early = d.wait_for_starting_new_tasks(reqs[:1500].copy(), 0.25)
    by: dict[int, list] = {}
    for j, g in enumerate(early):
        si = int(g["servant_index"])
        by.setdefault(si, []).append(RunningTask(j + 1, int(g["task_id"]), d.servant_location(si),
                                                 bytes(digests[(5000 - j) % n]).decode()))
    d.notify_servants_running_tasks([(d.servant_location(si), t) for si, t in by.items()])
    d.running_index_refresh()
    return w, reqs, src, keys, digests


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the record to this file")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "needs the GPU"
    rec = {"card": card(), "n": args.n}
    d = TaskDispatcher()
    assert d.backend == "cuda-sm90a"
    w, src_reqs, src, keys, digests = setup(d, args.n)
    n = args.n
    reqs = d.alloc_requests(n)
    reqs[...] = src_reqs
    out = d.alloc_grants(n)
    verdict = np.zeros(n, dtype=np.uint8)

    def pinned(a: np.ndarray) -> np.ndarray:  # both pipelines read their inputs from page-locked memory, as bench.py's
        buf = d._alloc(a.size, a.dtype).reshape(a.shape)
        buf[...] = a
        return buf

    pk, pd = pinned(keys), pinned(digests)
    src = TaskSources(pinned(src.args), pinned(src.args_offsets), pinned(src.args_index), pinned(src.source_digests))
    rec["args_strings"] = int(len(src.args_offsets) - 1)
    rec["args_bytes"] = int(src.args_offsets[-1])
    rec["args_len_min_max"] = [int(np.diff(src.args_offsets).min()), int(np.diff(src.args_offsets).max())]

    def one(kind: str, now: float):
        t0 = time.perf_counter()
        if kind == "descriptors":
            v, _, g = d.derive_filter_and_wait_for_starting_new_tasks(reqs, src, 3, now, out=out, verdict_out=verdict,
                                                                      want_hits=False)
        else:
            v, _, g = d.filter_and_wait_for_starting_new_tasks(reqs, pk, pd, now, out=out, verdict_out=verdict,
                                                               want_hits=False)
        dt = time.perf_counter() - t0
        st = d.last_solve_stats()
        res = (v.copy(), g["status"].copy(), g["servant_index"].copy())
        ok = g["status"] == STATUS_GRANTED
        d.free_tasks(g["task_id"][ok].copy())
        d.on_expiration_timer(now=now + 0.001)
        return dt, st, res

    times = {"descriptors": [], "keys": []}
    prep = {"descriptors": [], "keys": []}
    h2d = {}
    same = True
    for it in range(args.warmup + args.iters):
        got = {}
        for kind in (("descriptors", "keys") if it % 2 == 0 else ("keys", "descriptors")):
            dt, st, res = one(kind, 1.0 + 0.01 * it)
            got[kind] = res
            if it >= args.warmup:
                times[kind].append(1e3 * dt)
                prep[kind].append(st["prep_ms"])
            h2d[kind] = int(st["h2d_bytes"])
        a, b = got["descriptors"], got["keys"]
        same = same and all(x.shape == y.shape and (x == y).all() for x, y in zip(a, b))
    rec["pipelines_identical"] = bool(same)
    rec["offered"] = int((got["keys"][0] == 0).sum())
    for kind in times:
        rec[f"e2e_ms_{kind}"] = {"median": round(float(np.median(times[kind])), 4), "min": round(float(np.min(times[kind])), 4),
                                 "max": round(float(np.max(times[kind])), 4)}
        rec[f"prep_ms_{kind}"] = round(float(np.median(prep[kind])), 4)
        rec[f"h2d_bytes_{kind}"] = h2d[kind]
    rec["derive_ms_from_events"] = round(rec["prep_ms_descriptors"] - rec["prep_ms_keys"], 4)

    # the derivation kernel alone, both keys of every request, in a profiled phase of its own
    from torch.profiler import ProfilerActivity, profile

    for _ in range(args.warmup):
        d.derive_task_keys(reqs, src)
    calls = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            d.derive_task_keys(reqs, src)
        torch.cuda.synchronize()
    ks = [e for e in prof.key_averages() if "k_task_keys" in e.key]
    assert ks and ks[0].count == calls, [e.key for e in prof.key_averages()]
    dev_us = getattr(ks[0], "device_time", None) or ks[0].cuda_time  # average per call, microseconds
    rec["derive_kernel_ms"] = round(dev_us / 1e3, 4)
    rec["derive_Mkeys_per_s"] = round(2 * n / (dev_us / 1e6) / 1e6, 1)
    d.close()

    # the same keys on the host with the reference build (or the port where it was not built), one thread
    lib = ROOT / "oracle" / "_ref" / "libydref_keys.so"
    if not lib.exists():
        lib = ROOT / "checkers" / "libydport_keys.so"
    h = TaskDispatcher(str(lib))
    w.register(h, now=0.0, expires_in=3600.0)
    hreqs = w.build_requests(h)[:n].copy()
    assert (hreqs == src_reqs).all()
    t0 = time.perf_counter()
    hk, hd = h.derive_task_keys(hreqs, src)
    rec["host_derive_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    rec["host_backend"] = h.backend
    rec["host_keys_identical"] = bool((hk == keys).all() and (hd == digests).all())
    h.close()
    print(json.dumps(rec), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
