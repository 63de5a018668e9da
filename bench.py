#!/usr/bin/env python
"""bench.py -- task-assignment decisions/s on BASELINE.json's configs[1]
(100 k pending tasks x 2 k servants, 8 compiler digests, uniform slots).

A *step* is one pass of the hot path over one batch: the whole FIFO queue is offered to the
scheduler (n sequential WaitForStartingNewTask decisions, zero-wait).  Between steps, untimed,
the previous step's grants are freed (so every step starts from the same servant state), the
1 Hz expiration tick runs and L2 is flushed by writing a 256 MiB buffer.

  value   decisions/s with the request batch already resident in HBM (yd_stage_requests,
          untimed) when the timed region starts: CUDA events on the library's solve stream
          around everything between the upload and the grant download (yd_last_solve_stats).
  e2e     the same metric through the C-ABI call a scheduler front end makes
          (yd_wait_for_starting_new_tasks) with pinned HOST buffers: H2D of the requests, all
          kernels, D2H of the grants, host clock around the synchronous call.
  parity_in_run   the grants of this very process are compared with the reference's own
          TaskDispatcher (oracle/_ref, compiled verbatim; else the CPU restatement) on the same
          queue -- the whole queue for the 100 k configs, a stated prefix for the bigger ones --
          statuses, servant indices and task ids; a mismatch exits non-zero.
  roofline  `frac` = the compulsory bytes of one solve (requests in, grants + leases out, slot
          records, servant table) / the CUDA-event time / the HBM peak.  `model_frac` = SURVEY 8(d)'s
          matrix-row model (36*S + 32 B per decision: what the reference's O(S)-per-decision scan
          touches; this solver is O(1) per decision, so the model over-counts by design).
          `launch_bound` says what the limiter really is.
  workloads   sub-records for the other BASELINE configs (cfg2-random, cfg-self, cfg3, cfg4 =
          bloom + dedupe + solve, cfg5 on one GPU), each with value, e2e, cpu_baseline, parity.
  cpu_baseline  the reference's TaskDispatcher on a bounded sample of the same queue, one thread
          (the reference serialises every call on allocation_lock_).

`--impl reference` times that CPU implementation instead (rank 0 only).

N > 1 (torchrun, NCCL): ONE scheduler, ONE queue, range-sharded over the ranks: rank g holds the
g-th contiguous FIFO range in its HBM, the servant table is replicated, and the solve exchanges
the class tables (all-gather), per-class request counts (all-gather), the per-class request
prefixes the slots can reach (all-reduce of a disjointly written buffer) and the per-servant
claimed-slot counts (all-reduce) -- yadcc_b200/csrc/shard.cuh.  Strong scaling: the SAME problem at
every N.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

os.environ["NCCL_DEBUG"] = os.environ.get("YD_NCCL_DEBUG", "WARN")  # (NCCL's version banner goes to stdout: one JSON line only)

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from yadcc_b200 import STATUS_GRANTED, TaskDispatcher, pack_requests, unpack_grants  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402

METRIC = "task_assignment_decisions_per_sec"
UNIT = "decisions/s"
SUB_WORKLOADS = ["cfg2-random", "cfg-self", "cfg3", "cfg4", "cfg5"]
# decisions of the queue's head the CPU reference is run on (parity + cpu_baseline), sized for a few seconds each
CPU_SAMPLE = {"cfg1": 1000, "cfg2-mod": 100_000, "cfg2-random": 100_000, "cfg-self": 100_000, "cfg3": 100_000,
              "cfg4": 100_000, "cfg5": 50_000}


def build_workload(name: str, rank: int = 0):
    seed = 42 + 1000 * rank
    if name in ("cfg2-mod", "cfg4"):
        return S.config2(100_000, 2000, 8, seed=seed, variant="mod")
    if name == "cfg2-random":
        return S.config2(100_000, 2000, 8, seed=seed, variant="random")
    if name == "cfg1":
        return S.config1(seed=seed)
    if name == "cfg-self":
        return S.config_self(seed=seed)
    if name == "cfg3":
        return S.config3(1_000_000, 4000, 8, seed=seed)
    if name == "cfg5":  # BASELINE configs[4]: 10 M x 8 k
        return S.config5(10_000_000, 8000, 8, seed=seed)
    raise SystemExit(f"unknown workload {name}")


def workload_string(name: str, w) -> str:
    return f"{name}: {w.meta}"


def reference_library() -> tuple[Path, str]:
    ref = ROOT / "oracle" / "_ref" / "libydref.so"
    if ref.exists():
        return ref, "reference"
    ref = ROOT / "oracle" / "libydoracle.so"
    if not ref.exists():
        subprocess.check_call(["make", "-C", str(ROOT / "oracle"), "libydoracle.so"])
    return ref, "port"


class ClockSampler(threading.Thread):
    """nvidia-smi clocks + throttle reasons during the timed region (rank 0 only)."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        super().__init__(daemon=True)
        self.index = index
        self.rows: list[list[str]] = []
        self.stop_flag = threading.Event()

    def run(self):
        while not self.stop_flag.is_set():
            try:
                out = subprocess.run(
                    ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                    capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.splitlines()[0].split(",")])
            except Exception:
                pass
            self.stop_flag.wait(0.25)

    def summary(self) -> dict:
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        sm = sorted(float(r[1]) for r in self.rows if r[1].replace(".", "").isdigit())
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            for k, nm in enumerate(names):
                if len(r) > 5 + k and r[5 + k].lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None,
                "sm_max_mhz": float(self.rows[0][2]) if self.rows[0][2].replace(".", "").isdigit() else None,
                "samples": len(self.rows), "reasons": sorted(reasons)}


def measured_hbm_peak() -> tuple[float, str]:
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        try:
            return float(json.loads(p.read_text())["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "data sheet (H100 SXM HBM3, 3.35 TB/s)"


# ---------------------------------------------------------------------------------------------
# the reference on the host
# ---------------------------------------------------------------------------------------------

class Cfg4Stages:
    """BASELINE configs[3]: the 6124-TU LLVM-11 trace looped to 100 k requests with the cache bloom filter on.
    Stage 1: requests whose cache key may be cached are dropped (distributed_cache_reader.cc:70-77); stage 2:
    requests whose task digest is already being compiled join that task (running_task_keeper.cc:67-75); stage 3:
    the rest is solved as config 2.  Same code for the CUDA library and the CPU reference."""

    def __init__(self, d: TaskDispatcher, w, n: int):
        rng = np.random.default_rng(46)
        self.keys = ["yadcc-cxx2-entry-" + rng.bytes(32).hex() for _ in range(6124)]
        r2 = np.random.default_rng(11)
        digests = [r2.bytes(32).hex() for _ in range(6124)]
        r3 = np.random.default_rng(4)
        cached = [k for k, m in zip(self.keys, r3.random(len(self.keys)) < 0.3) if m]
        tu = np.arange(n) % len(self.keys)
        km = TaskDispatcher._key_matrix(self.keys)       # (6124, 81) bytes
        dm = TaskDispatcher._key_matrix(digests)         # (6124, 64) bytes
        # the queue's cache keys / task digests as byte matrices, in pinned host memory when the backend has it
        self.trace = self._pinned(d, km[tu])
        self.trace_digests = self._pinned(d, dm[tu])
        self.d = d
        d.bloom_reset()
        d.bloom_add(cached)
        # an earlier wave is still compiling: its servants list those tasks in their heartbeats
        from yadcc_b200 import RunningTask

        reqs = w.build_requests(d)
        early = d.wait_for_starting_new_tasks(reqs[:1500].copy(), 0.25)
        locs = [d.servant_location(i) for i in range(len(w.servants))]
        by_servant: dict[int, list] = {}
        for j, gr in enumerate(early):
            by_servant.setdefault(int(gr["servant_index"]), []).append(
                RunningTask(j + 1, int(gr["task_id"]), locs[int(gr["servant_index"])], digests[5000 - j]))
        d.notify_servants_running_tasks([(locs[si], tasks) for si, tasks in by_servant.items()])
        d.running_index_refresh()
        self.early_ids = early["task_id"].copy()

    @staticmethod
    def _pinned(d: TaskDispatcher, m: np.ndarray) -> np.ndarray:
        try:
            buf = d._alloc(m.size, np.dtype(np.uint8)).reshape(m.shape)
            buf[...] = m
            return buf
        except Exception:
            return np.ascontiguousarray(m)

    def filter(self, reqs: np.ndarray) -> np.ndarray:
        n = len(reqs)
        hit = self.d.bloom_possibly_contains(self.trace[:n])
        joined = self.d.find_running_tasks(self.trace_digests[:n])
        return reqs[~hit.astype(bool) & (joined["found"] == 0)]

    def one_call(self, reqs: np.ndarray, now: float, out: np.ndarray):
        """The three stages as ONE C-ABI call (yd_filter_and_wait_for_starting_new_tasks): (grants, offered)."""
        n = len(reqs)
        if getattr(self, "verdict", None) is None or len(self.verdict) < n:
            self.verdict = self._pinned(self.d, np.zeros(n, dtype=np.uint8))
        _, _, g = self.d.filter_and_wait_for_starting_new_tasks(reqs, self.trace[:n], self.trace_digests[:n], now, out=out,
                                                                verdict_out=self.verdict, want_hits=False)
        return g, len(g)


def cpu_reference_sample(name: str, n_sample: int):
    """The reference on the head of the workload's queue: (kind, grants, seconds, decisions)."""
    lib, kind = reference_library()
    w = build_workload(name)
    d = TaskDispatcher(str(lib))
    w.register(d, now=0.0, expires_in=3600.0)
    reqs = w.build_requests(d)[:n_sample]
    t0 = time.perf_counter()
    if name == "cfg4":
        st = Cfg4Stages(d, w, len(reqs))
        t0 = time.perf_counter()  # (the stage set-up is state, not the timed pass)
        kept = st.filter(reqs)
        g = d.wait_for_starting_new_tasks(kept, 1.5)
    else:
        g = d.wait_for_starting_new_tasks(reqs, 1.5)
    dt = time.perf_counter() - t0
    out = g.copy()
    d.close()
    return kind, out, dt, len(reqs)


def grants_equal(a: np.ndarray, b: np.ndarray) -> bool:
    """Statuses, servants and task ids (relative to the first id each side handed out)."""
    if a.shape != b.shape or not (a["status"] == b["status"]).all() or not (a["servant_index"] == b["servant_index"]).all():
        return False
    ok = a["status"] == STATUS_GRANTED
    if not ok.any():
        return True
    ia, ib = a["task_id"][ok].astype(np.int64), b["task_id"][ok].astype(np.int64)
    return bool(((ia - ia[0]) == (ib - ib[0])).all())


# ---------------------------------------------------------------------------------------------
# one workload on the GPU
# ---------------------------------------------------------------------------------------------

def measure_workload(name: str, dev_index: int, steps: int, warmup: int, solver: int, with_cpu: bool, flush, sampler=None):
    import torch

    w = build_workload(name)
    d = TaskDispatcher(device=dev_index, solver=solver)
    assert d.backend == "cuda-sm90a"
    w.register(d, now=0.0, expires_in=3600.0)
    src = w.build_requests(d)
    stages = Cfg4Stages(d, w, len(src)) if name == "cfg4" else None
    n = len(src)
    S_count = len(w.servants)
    reqs = d.alloc_requests(n)  # pinned host memory
    out = d.alloc_grants(n)
    reqs[...] = src
    reqs16 = d.alloc_requests16(n)  # the packed interface's buffers (16 B up, 8 B down), pinned too
    out8 = d.alloc_grants8(n)
    pack_requests(src, reqs16)
    use_packed = stages is None  # (cfg4's queue is filtered on the way: it goes through the plain call)
    if os.environ.get("BENCH_NO_PACKED"):  # (diagnostics: time the plain call alone, as before the packed interface existed)
        use_packed = False

    def one_pass(queue, now, mode):
        """(grants, decisions offered to the solver); mode: "staged" | "plain" | "packed" """
        if stages is not None and mode != "three-calls":
            return stages.one_call(reqs[: len(queue)], now, out)  # bloom + dedupe + solve, one call, queue in pinned memory
        if stages is not None:
            queue = stages.filter(queue)
            buf = reqs[: len(queue)]
            buf[...] = queue
            queue = buf
        if mode == "staged":
            d.stage_requests(queue)
            return d.wait_for_staged_tasks(len(queue), now, out=out), len(queue)
        if mode == "packed":
            g8, ids = d.wait_for_starting_new_tasks_packed(reqs16[: len(queue)], now, out8=out8, unpack=False)
            return (g8, ids), len(queue)
        return d.wait_for_starting_new_tasks(queue, now, out=out), len(queue)

    # ---- parity in this run: the reference on the head of the same queue -------------------------------
    parity, cpu = None, None
    if with_cpu:
        n_s = min(n, CPU_SAMPLE[name])
        kind, g_cpu, cpu_s, _ = cpu_reference_sample(name, n_s)
        head = src[:n_s].copy()
        g_gpu, _ = one_pass(head, 1.5, "plain")
        parity = grants_equal(g_gpu.copy(), g_cpu)
        d.free_tasks(g_gpu["task_id"][g_gpu["status"] == STATUS_GRANTED].copy())
        d.on_expiration_timer(now=1.6)
        if use_packed:  # the same head through the packed interface (the call `e2e` is timed on)
            (g8, ids), _ = one_pass(head, 1.7, "packed")
            g_gpu = unpack_grants(g8.copy(), ids)
            parity = parity and grants_equal(g_gpu, g_cpu)
            d.free_tasks(g_gpu["task_id"][g_gpu["status"] == STATUS_GRANTED].copy())
            d.on_expiration_timer(now=1.8)
        cpu = {"value": n_s / cpu_s, "unit": UNIT, "cores": 1, "kind": kind,
               "sample": f"the first {n_s} of the queue's {n} requests, once ({cpu_s:.2f} s), single thread; the reference "
                         f"serialises on allocation_lock_ (host has {os.cpu_count()} cores)"}
        reqs[...] = src

    dev_ms, e2e_ms, e2e24_ms, launches, n_solves = [], [], [], 0, 0
    granted = h2d = d2h = h2d24 = d2h24 = solver_used = offered = 0
    prev_ids = None
    t_wall0 = time.perf_counter()
    for it in range(warmup + steps):
        now = 2.0 + it
        if prev_ids is not None:
            d.free_tasks(prev_ids)
        d.on_expiration_timer(now=now)
        flush.fill_(it & 0xFF)
        if it == warmup:
            torch.cuda.synchronize()
            if sampler is not None:
                sampler.start()
            t_wall0 = time.perf_counter()
        torch.cuda.synchronize()
        # -- timed (e2e): HOST buffers --------------------------------------------------------------
        t0 = time.perf_counter()
        g, offered = one_pass(src if stages is not None else reqs, now, "packed" if use_packed else "plain")
        t1 = time.perf_counter()
        st = d.last_solve_stats()
        if use_packed:
            g = unpack_grants(g[0], g[1])  # (untimed: the caller's id arithmetic, done here for the FreeTask below)
        ok = g["status"] == STATUS_GRANTED
        prev_ids = g["task_id"][ok].copy()
        granted = int(ok.sum())
        if it >= warmup:
            e2e_ms.append(1e3 * (t1 - t0))
            launches += st["kernel_launches"]
            n_solves += 1
            h2d, d2h = st["h2d_bytes"], st["d2h_bytes"]
            solver_used = st["solver"]
        if use_packed and n <= 2_000_000:
            # -- timed (e2e, 24-byte requests / 16-byte grants): the plain call, for comparison -----------------
            # (not for the 10 M queue: as the sixth workload of one process this third pass timed several times
            # slower than the same call alone in a fresh process; a harness artefact, not traced further)
            d.free_tasks(prev_ids)
            d.on_expiration_timer(now=now)
            flush.fill_((it + 7) & 0xFF)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g, _ = one_pass(reqs, now, "plain")
            t1 = time.perf_counter()
            st = d.last_solve_stats()
            ok = g["status"] == STATUS_GRANTED
            prev_ids = g["task_id"][ok].copy()
            assert int(ok.sum()) == granted
            if it >= warmup:
                e2e24_ms.append(1e3 * (t1 - t0))
                h2d24, d2h24 = st["h2d_bytes"], st["d2h_bytes"]
        # -- timed (value): the queue already resident in HBM ---------------------------------------------
        d.free_tasks(prev_ids)
        d.on_expiration_timer(now=now)
        flush.fill_(~it & 0xFF)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g, _ = one_pass(src if stages is not None else reqs, now, "staged")
        t1 = time.perf_counter()
        st = d.last_solve_stats()
        ok = g["status"] == STATUS_GRANTED
        prev_ids = g["task_id"][ok].copy()
        assert int(ok.sum()) == granted
        last_grants = g.copy()
        if it >= warmup:
            # CUDA events on the solve stream (cfg4: the filter stages' kernels + compaction are in prep_ms, the uploads
            # of keys / digests / queue are not: `value` counts from "inputs resident in HBM")
            dev_ms.append(st["prep_ms"] + st["solve_ms"] + st["final_ms"])
            launches += st["kernel_launches"]
            n_solves += 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t_wall0
    d.free_tasks(prev_ids)
    d.close()
    K = len(dev_ms)
    ms_step = sum(dev_ms) / K
    e2e_step = sum(e2e_ms) / K
    decisions = n  # the queue offered per step (cfg4: before its pre-filter stages)
    rec = {
        "workload": workload_string(name, w) + (" + bloom pre-filter (30 % of 6124 TU keys cached) + in-flight task dedupe"
                                                if name == "cfg4" else ""),
        "decisions_per_step": decisions, "granted_per_step": granted, "solver_decisions_per_step": offered,
        "value": decisions / (ms_step / 1e3), "unit": UNIT, "ms_per_step": ms_step, "steps": K,
        "e2e": {"value": decisions / (e2e_step / 1e3), "unit": UNIT, "ms_per_step": e2e_step,
                "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
                "call": "yd_wait_for_starting_new_tasks_packed (16-byte requests, 8-byte grants)" if use_packed
                        else "yd_filter_and_wait_for_starting_new_tasks (bloom + in-flight dedupe + solve in one call)"},
        "gpu_launches_per_step": launches // max(1, n_solves),
        "solver": {1: "row-scan", 2: "slot-stream"}.get(solver_used, str(solver_used)),
        "parity_in_run": parity, "cpu_baseline": cpu,
    }
    if e2e24_ms:
        e24 = sum(e2e24_ms) / len(e2e24_ms)
        rec["e2e_unpacked"] = {"value": decisions / (e24 / 1e3), "unit": UNIT, "ms_per_step": e24,
                               "h2d_bytes_per_step": int(h2d24), "d2h_bytes_per_step": int(d2h24),
                               "call": "yd_wait_for_starting_new_tasks (24-byte requests, 16-byte grants)"}
    extra = {"e2e_ms": e2e_ms, "dev_ms": dev_ms, "launches": launches, "n_solves": n_solves, "wall": wall,
             "S": S_count, "n": n, "w": w, "last_grants": last_grants}
    return rec, extra


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir: str, grants: np.ndarray) -> None:
    """The grants of the last timed step as float64 arrays, one file per field.  Above DUMP_LIMIT_BYTES a fixed
    seeded sample of the grants is written instead, with its indices into the batch (sample_index.npy)."""
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    fields = ("status", "servant_index", "task_id")
    idx = np.arange(len(grants))
    if len(grants) * 8 * (len(fields) + 1) > DUMP_LIMIT_BYTES:
        keep = DUMP_LIMIT_BYTES // (8 * (len(fields) + 1))
        idx = np.sort(np.random.default_rng(0).choice(len(grants), size=keep, replace=False))
        np.save(d / "sample_index.npy", idx.astype(np.float64))
    for f in fields:
        np.save(d / f"grants_{f}.npy", grants[f][idx].astype(np.float64))  # (task ids stay below 2**53)


def latency_sweep(dev_index: int, sizes=(1, 32, 1024), reps=200):
    """Dispatch latency = the whole C-ABI call (enqueue -> grant available to the caller), pinned host buffers."""
    d = TaskDispatcher(device=dev_index)
    w = build_workload("cfg2-mod")
    w.register(d, now=0.0, expires_in=3600.0)
    src = w.build_requests(d)
    rows = []
    for n in sizes:
        reqs = d.alloc_requests(n)
        reqs[...] = src[:n]
        out = d.alloc_grants(n)
        ts = []
        for it in range(reps + 5):
            t0 = time.perf_counter()
            g = d.wait_for_starting_new_tasks(reqs, 1.0 + it, out=out)
            t1 = time.perf_counter()
            d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED].copy())
            if it >= 5:
                ts.append(1e3 * (t1 - t0))
        ts = np.sort(np.asarray(ts))
        rows.append({"batch": n, "p50_ms": round(float(ts[len(ts) // 2]), 4), "p99_ms": round(float(ts[int(len(ts) * 0.99)]), 4)})
    d.close()
    return rows


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return  # other ranks exit 0 without work
    lib, kind = reference_library()
    w = build_workload(args.workload)
    d = TaskDispatcher(str(lib))
    w.register(d, now=0.0, expires_in=3600.0)
    reqs_all = w.build_requests(d)
    n_all = len(reqs_all)
    # a bounded sample per step so that the whole run ends within a few minutes (~15 us per decision)
    n = min(n_all, max(1000, int(120.0 / max(1, args.steps + args.warmup) / 15e-6)))
    reqs = reqs_all[:n]
    times, granted = [], 0
    for it in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        g = d.wait_for_starting_new_tasks(reqs, 0.001)
        t1 = time.perf_counter()
        ok = g["status"] == STATUS_GRANTED
        granted = int(ok.sum())
        d.free_tasks(g["task_id"][ok])
        d.on_expiration_timer(now=1.0 + it)
        if it >= args.warmup:
            times.append(t1 - t0)
    d.close()
    total = sum(times)
    value = n * len(times) / total
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * total / len(times), "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "f64", "data": "synthetic", "impl": "reference",
        "config": {"workload": workload_string(args.workload, w), "decisions_per_step": n_all, "sampled_decisions_per_step": n,
                   "granted_per_sampled_step": granted},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": 1, "kind": kind,
                         "sample": f"{len(times)} steps x the first {n} of the queue's {n_all} requests, single thread "
                                   f"(the reference serialises on allocation_lock_), host has {os.cpu_count()} cores"},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


def run_ours(args):
    import torch

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        from bench_sharded import run_sharded  # the range-sharded scheduler over NCCL

        return run_sharded(args, rank, world, local)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the H100's 50 MB L2
    sampler = ClockSampler(local)
    rec, ex = measure_workload(args.workload, local, args.steps, args.warmup, args.solver, not args.no_cpu_baseline, flush, sampler)
    sampler.stop_flag.set()
    sampler.join(timeout=2)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, ex["last_grants"])
    if rec["parity_in_run"] is False:
        print(json.dumps({"error": "parity_in_run failed", "workload": args.workload}), file=sys.stderr)

    subs = {}
    if args.sub != "none" and args.workload == "cfg2-mod":
        names = SUB_WORKLOADS if args.sub == "all" else [x for x in args.sub.split(",") if x]
        for name in names:
            r2, _ = measure_workload(name, local, args.sub_steps, 3, args.solver, not args.no_cpu_baseline, flush)
            subs[name] = r2
    lat = latency_sweep(local) if args.workload == "cfg2-mod" and not args.no_latency else None

    peak, peak_src = measured_hbm_peak()
    n, S_count, ms_step = ex["n"], ex["S"], rec["ms_per_step"]
    model_bytes = 36 * S_count + 32  # SURVEY.md 8(d) matrix-row model, per decision
    # what one staged solve has to move at the very least: requests in (24 B), grants out (16 B), one lease per grant
    # (16 B), the kept slot order's records (8 B per slot), one servant-table read
    slots = int(sum(min(sv.num_processors, sv.max_tasks) for sv in ex["w"].servants))
    compulsory = 24 * n + 16 * n + 16 * rec["granted_per_step"] + 8 * slots + 36 * S_count
    e2e_ms = ex["e2e_ms"]
    line = {
        "metric": METRIC, "value": rec["value"], "unit": UNIT, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "u32", "data": "synthetic",
        "config": {"workload": workload_string(args.workload, ex["w"]), "decisions_per_step": n,
                   "granted_per_step": rec["granted_per_step"], "parallelism": "1 GPU",
                   "l2": "flushed between steps (256 MiB write)", "solver": rec["solver"],
                   "between_steps_untimed": "FreeTask of the previous grants + OnExpirationTimer tick"},
        "e2e": rec["e2e"],
        "e2e_unpacked": rec.get("e2e_unpacked"),
        "gpu_launches": int(ex["launches"]),
        "parity_in_run": rec["parity_in_run"],
        "roofline": {
            "bound": "hbm",
            "kernel": ("k_fused_front (fused.cuh): the whole solve as ONE persistent launch, one 1024-thread block per SM, two grid barriers"
                       if rec["gpu_launches_per_step"] == 1 else
                       f"{rec['solver']} solve pipeline (one CUDA graph, {rec['gpu_launches_per_step']} kernels)"),
            # achieved = ALGORITHMIC (compulsory) bytes per launch / the launch's duration, CUDA events on the solve stream
            "achieved": compulsory / (ms_step / 1e3) / 1e9, "peak": peak, "unit": "GB/s",
            "frac": compulsory / (ms_step / 1e3) / 1e9 / peak,
            "peak_source": peak_src, "kernel_ms_per_step": ms_step,
            "model_frac": n * model_bytes / (ms_step / 1e3) / 1e9 / peak, "algorithmic_bytes_per_decision_model": model_bytes,
            "compulsory": {"bytes_per_step": compulsory, "frac": compulsory / (ms_step / 1e3) / 1e9 / peak},
            "launch_bound": {"kernels": rec["gpu_launches_per_step"], "graph_us": 1e3 * ms_step},
            "note": "achieved/frac = compulsory bytes of one solve (requests in, grants + leases out, slot records, servant "
                    "table: `compulsory`) / CUDA-event time of the launch / HBM peak. "
                    "model_frac is SURVEY 8(d)'s 36*S+32 B per decision (the reference's "
                    "O(S) scan per decision; this solver does O(1) work per decision, so it exceeds 1). The solve is bound by "
                    "the dependent-latency chain of its phases (two grid barriers, index chasing through L2), not by "
                    "bandwidth: DESIGN.md section 5.",
        },
        "cpu_baseline": rec["cpu_baseline"],
        "workloads": subs,
        "cfg5_strong": subs.get("cfg5"),  # the N = 1 point of the strong-scaling curve the N > 1 lines carry
        "dispatch_latency": lat,
        "clocks": sampler.summary(),
        "wall_s_timed_loop": ex["wall"],
        "e2e_ms_steps": {"min": round(min(e2e_ms), 4), "median": round(sorted(e2e_ms)[len(e2e_ms) // 2], 4),
                         "max": round(max(e2e_ms), 4)},
        "latency_ms": {"p50": float(np.percentile(e2e_ms, 50)), "p99": float(np.percentile(e2e_ms, 99)),
                       "what": "enqueue->grant for every request of the 100 k batch (whole-batch call); "
                               "dispatch_latency has the small-batch figures"},
    }
    print(json.dumps(line))
    bad = [k for k, v in [(args.workload, rec)] + list(subs.items()) if v["parity_in_run"] is False]
    if bad:
        print(f"bench.py: parity_in_run FAILED for {bad}", file=sys.stderr)
        sys.exit(3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="cfg2-mod")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-latency", action="store_true")
    ap.add_argument("--solver", type=int, default=0, help="0 auto, 1 row-scan, 2 slot-stream")
    ap.add_argument("--sub", default="all", help="sub-records beside the headline: all | none | comma-separated workloads")
    ap.add_argument("--sub-steps", type=int, default=5)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the grants of the headline workload's last timed step to DIR/*.npy (float64)")
    args = ap.parse_args()
    if args.warmup < 3:
        args.warmup = 3
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
