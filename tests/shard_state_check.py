#!/usr/bin/env python
"""State handover of the range-sharded scheduler (yd_shard_export_state / yd_shard_import_state, include/ydshard.h) on
ONE GPU: W rank handles in W threads of one process over the test-only NCCL stand-in, as in shard_threads_check.py
(imported first: it loads tests/fake_nccl/libnccl.so.2 with RTLD_GLOBAL; this process must not import torch).

The checker is ONE scheduler fed the concatenated queue and never stopped: the port's state build
(checkers/libydport_state.so), or -- at scale -- a single CUDA handle.  Every handle pre-interns the streams' servant
digests and IP prefixes, so that the exports of all backends are byte-comparable (ydstate.h).  At seeded cuts of a
stream:
  export     every rank's export is the same bytes, equal to the checker's
  continue   --mode export: the same group plays on (the export changed nothing)
             --mode handover: the export goes into a fresh group of the next size of --targets (0: one plain CUDA
             handle, yd_import_state), which plays the rest of the stream
After every event the harness of shard_threads_check.py compares grants, servant state, next id, lease counts,
keep-alive answers and running tasks with the checker's; at the end the exports are compared once more.

Prints one JSON line per case and a final {"shard_state": ...} line; exit code 0 iff everything matched.
"""
import argparse
import ctypes as C
import json
import sys
import time

_argv, sys.argv = sys.argv, sys.argv[:1]
import shard_threads_check as T  # noqa: E402  (loads the NCCL stand-in before anything else)
sys.argv = _argv

import numpy as np  # noqa: E402

from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200.dispatcher import Servant, StateError, TaskDispatcher  # noqa: E402

PORT_STATE = T.ROOT / "checkers" / "libydport_state.so"
ZOMBIE = 2  # YD_STATE_LEASE_ZOMBIE


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--fuzz", default="", help="comma-separated fuzz_stream seeds")
    ap.add_argument("--mode", choices=["export", "handover"], default="export")
    ap.add_argument("--targets", default="1,2,3,4,0", help="group sizes the handovers go to, in turn (0: a plain handle)")
    ap.add_argument("--cuts", type=int, default=5)
    ap.add_argument("--scale", default="", help="comma-separated: cfg2-mod, 1m")
    ap.add_argument("--refusals", action="store_true")
    ap.add_argument("--seed", type=int, default=0)
    return ap.parse_args()


def pre_intern(d: TaskDispatcher, stream: S.Stream) -> None:
    """Intern every digest servants report and every servant IP prefix, in stream order (ydstate.h: the CUDA backend
    interns them on its own, the port does not)."""
    for ev in stream.events:
        if ev[0] == "hb":
            sv: Servant = ev[2]
            for e in sv.environments:
                d.intern_env(e)
            loc = sv.observed_location
            for k, c in enumerate(loc):
                if c == ":":
                    d.intern_ip(loc[:k])


def event_time(ev):
    return ev[1] if ev[0] in ("hb", "solve", "wait", "keepalive", "tick") else None


def shard_export(lib, ranks, now: float) -> list:
    """The collective export on every rank: the size query, then the bytes."""
    t = T.ns(now)
    sizes = T.par([lambda d=d: lib.yd_shard_export_state(d._h, t, None, 0) for d in ranks])
    bufs = [C.create_string_buffer(max(n, 1)) for n in sizes]
    got = T.par([lambda d=d, b=b, n=n: lib.yd_shard_export_state(d._h, t, b, n) for d, b, n in zip(ranks, bufs, sizes)])
    assert got == sizes, (got, sizes)
    return [b.raw[:n] for b, n in zip(bufs, sizes)]


def shard_import(lib, ranks, blobs, now: float) -> list:
    t = T.ns(now)
    return T.par([lambda d=d, b=b: lib.yd_shard_import_state(d._h, t, b, len(b)) for d, b in zip(ranks, blobs)])


def new_group(lib, world: int, **cfg) -> list:
    ranks = [TaskDispatcher(lib, **cfg) for _ in range(world)]
    uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
    assert lib.yd_shard_unique_id(uid) == 0
    assert T.par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, world, uid) for r in range(world)]) == [0] * world
    return ranks


def close_group(lib, ranks) -> None:
    for d in ranks:
        lib.yd_shard_finalize(d._h)
        d.close()


def fake_stats(world: int) -> np.ndarray:
    """The stand-in's per-rank counters: collectives, all-gathers, all-reduces, bytes."""
    out = []
    for r in range(world):
        a = (C.c_ulonglong * 4)()
        T.FAKE.yd_fake_nccl_stats(r, a)
        out.append(list(a))
    return np.asarray(out, dtype=np.int64)


def is_fresh(d: TaskDispatcher) -> bool:
    return d.num_servants() == 0 and d.next_task_id() == 0 and d.num_tasks() == 0 and not d.get_running_tasks()


class StateHarness(T.Harness):
    """shard_threads_check's harness over a group that can be replaced by the group (or plain handle) an export was
    imported into."""

    def __init__(self, name: str, world: int, seed: int, checker: TaskDispatcher):
        self.name, self.W = name, world
        self.rng = np.random.default_rng(seed)
        self.lib = _abi.load_library()
        self.ranks = new_group(self.lib, world)
        self.oracle = checker
        self.plain = False
        self.pending = np.zeros(0, dtype=_abi.REQ_DTYPE)
        self.outstanding: dict[int, int] = {}
        self.counts = {"events": 0, "solves": 0, "frees": 0, "collectives": 0, "handbacks": 0, "retried": 0,
                       "max_merge_rounds": 0, "lazy_checks": 0, "cuts": 0, "handovers": 0, "zombie_cuts": 0,
                       "split_lease_cuts": 0, "split_group_cuts": 0, "export_s": [], "import_s": []}
        self.cuts: list = []
        self.ev = None

    def close(self):
        if self.plain:
            self.ranks[0].close()
        else:
            close_group(self.lib, self.ranks)

    # a plain handle (W = 1, no sharded calls) after a handover to yd_import_state
    def solve(self, now, full):
        if not self.plain:
            return super().solve(now, full)
        g = self.ranks[0].wait_for_starting_new_tasks(np.ascontiguousarray(full), now).copy()
        g1 = self.oracle.wait_for_starting_new_tasks(np.ascontiguousarray(full), now).copy()
        for f in ("status", "servant_index", "task_id"):
            if not (g[f] == g1[f]).all():
                self.fail("grants differ", field=f)
        self.counts["solves"] += 1
        ok = g["status"] == _abi.STATUS_GRANTED
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        return g

    def free(self, ids):
        if not self.plain:
            return super().free(ids)
        ids = np.asarray(ids, dtype=np.uint64)
        self.ranks[0].free_tasks(ids)
        self.oracle.free_tasks(ids)
        self.counts["frees"] += 1
        for i in ids.tolist():
            self.outstanding.pop(i, None)

    def export(self, now: float) -> bytes:
        t0 = time.perf_counter()
        if self.plain:
            blobs = [self.ranks[0].export_state(now)]
        else:
            blobs = shard_export(self.lib, self.ranks, now)
        self.counts["export_s"].append(time.perf_counter() - t0)
        if any(b != blobs[0] for b in blobs):
            self.fail("ranks exported different bytes", sizes=[len(b) for b in blobs])
        want = self.oracle.export_state(now)
        if blobs[0] != want:
            self.fail("export differs from the single scheduler's", sharded=len(blobs[0]), single=len(want))
        return blobs[0]

    def cover(self, blob: bytes) -> None:
        """What the cut carries: a zombie lease, leases on two ranks, a bookkeeper group held by two ranks."""
        self.counts["cuts"] += 1
        if self.plain:
            return
        held = [d.num_tasks() for d in self.ranks]
        self.counts["split_lease_cuts"] += sum(x > 0 for x in held) >= 2
        owners: dict[str, set] = {}
        for r, d in enumerate(self.ranks):
            for t in d.get_running_tasks():
                owners.setdefault(t.servant_location, set()).add(r)
        self.counts["split_group_cuts"] += any(len(v) >= 2 for v in owners.values())
        hdr = parse_leases(blob)
        self.counts["zombie_cuts"] += bool((hdr["flags"] & ZOMBIE).any())

    def hand_over(self, blob: bytes, now: float, target: int) -> None:
        old, old_plain = self.ranks, self.plain
        t0 = time.perf_counter()
        if target == 0:
            d = TaskDispatcher(self.lib)
            d.import_state(blob, now=now)
            ranks = [d]
        else:
            ranks = new_group(self.lib, target)
            rcs = shard_import(self.lib, ranks, [blob] * target, now)
            if rcs != [_abi.STATE_OK] * target:
                self.fail("import refused", rcs=rcs)
        self.counts["import_s"].append(time.perf_counter() - t0)
        if old_plain:
            old[0].close()
        else:
            close_group(self.lib, old)
        self.ranks, self.W, self.plain = ranks, max(target, 1), target == 0
        self.counts["handovers"] += 1


def parse_leases(blob: bytes) -> np.ndarray:
    """The lease records of an export (ydstate.h), located by walking the sections before them."""
    import struct

    at = 32

    def u32():
        nonlocal at
        v = struct.unpack_from("<I", blob, at)[0]
        at += 4
        return v

    def skip_str():
        nonlocal at
        n = u32()
        at += n

    for _ in range(2):
        for _ in range(u32()):
            skip_str()
    for _ in range(u32()):
        at += 56  # version .. ever_assigned_tasks
        skip_str()
        skip_str()
        for _ in range(u32()):
            skip_str()
    n = struct.unpack_from("<Q", blob, at)[0]
    return np.frombuffer(blob, dtype=[("id", "<u8"), ("servant", "<u4"), ("flags", "<u4"), ("rel", "<i8")], count=n,
                         offset=at + 8)


def play(h: StateHarness, streams, cuts, mode: str, targets) -> None:
    """Events of the checker's stream (streams[-1]), with an export -- and in handover mode a handover -- at each cut."""
    base = streams[-1]
    now, k_target = 0.0, 0
    for k, ev in enumerate(base.events):
        if k in cuts:
            blob = h.export(now)
            h.cover(blob)
            if mode == "handover":
                h.hand_over(blob, now, targets[k_target % len(targets)])
                k_target += 1

        def build(f, k=k):
            vals = [f(d) for d in h.ranks] + [f(h.oracle)]
            for v in vals[:-1]:
                assert v.shape == vals[-1].shape and (v == vals[-1]).all(), "intern ids differ between handles"
            return vals[-1]
        h.event(ev, build)
        t = event_time(ev)
        now = t if t is not None else now
    h.export(now)  # the final exports


def fuzz_case(seed: int, world: int, mode: str, targets, n_cuts: int, case_seed: int):
    checker = TaskDispatcher(str(PORT_STATE))
    h = StateHarness(f"fuzz-{seed}", world, case_seed, checker)
    make = lambda d: S.fuzz_stream(d, seed, n_servants=8 + seed % 30)  # noqa: E731
    ok = True
    try:
        streams = [make(d) for d in h.ranks + [checker]]
        for d, st in zip(h.ranks + [checker], streams):
            pre_intern(d, st)
        n = len(streams[-1].events)
        cuts = set(int(x) for x in np.random.default_rng(case_seed).choice(np.arange(1, n), min(n_cuts, n - 1),
                                                                           replace=False))
        play(h, streams, cuts, mode, targets)
    except T.Mismatch:
        ok = False
    finally:
        h.close()
        checker.close()
    return h, ok


def million_workload() -> S.Workload:
    """4 k servants with 256 free slots each; 1 M requests fill them all."""
    servants = [Servant(f"{S.servant_ip(k)}:8335", environments=["e" * 64], num_processors=256, max_tasks=256,
                        priority=1 + k % 2) for k in range(4000)]
    return S.Workload("1m", servants, ["e" * 64],
                      lambda d: d.make_requests(1_000_000, "e" * 64, "172.16.0.1", expires_in=30))


def scale_case(name: str, world: int):
    """The group's export equals a single CUDA handle's (the checker) after the first solve; a handover into a fresh
    group continues identically, and the final exports agree."""
    w = T.CONFIGS["cfg2-mod"]() if name == "cfg2-mod" else million_workload()
    checker = TaskDispatcher(_abi.load_library())
    h = StateHarness(name, world, 5, checker)
    ok = True
    try:
        streams = [T.workload_stream(w, d) for d in h.ranks + [checker]]
        ev = streams[-1].events
        first = next(i for i, e in enumerate(ev) if e[0] == "wait") + 1
        play(h, streams, {first, first + 2}, "handover", [world])
    except T.Mismatch:
        ok = False
    finally:
        h.close()
        checker.close()
    return h, ok


def refusal_case(world: int):
    """Refusals come back with the same code on every rank and leave every rank fresh; a retry then succeeds.  A single
    handle's export is what the group loads.  The single-handle calls refuse sharded handles."""
    lib = _abi.load_library()
    src = TaskDispatcher(lib)
    other = TaskDispatcher(lib, servant_min_memory_for_accepting_new_task="1G")
    ok, line = True, {"case": "refusals", "world": world}
    groups = []
    try:
        for d in (src, other):
            for k in range(6):
                d.keep_servant_alive(Servant(f"10.8.0.{k}:8000", environments=["ab" * 32], num_processors=8, max_tasks=8),
                                     100.0, now=0.0)
            r = d.make_requests(30, "ab" * 32, "172.16.0.1", expires_in=30)
            d.wait_for_starting_new_tasks(r, now=1.0)
        blob, wrong = src.export_state(now=2.0), other.export_state(now=2.0)
        stats0 = fake_stats(world)

        dirty = new_group(lib, world)
        groups.append(dirty)
        dirty[1].keep_servant_alive(Servant("10.8.1.1:8000", environments=["ab" * 32]), 10.0, now=0.0)
        got = {"not-fresh": shard_import(lib, dirty, [blob] * world, 2.0)}
        fresh_after = [is_fresh(d) for i, d in enumerate(dirty) if i != 1]

        g = new_group(lib, world)
        groups.append(g)
        differs = [blob] * world
        differs[1] = src.export_state(now=3.0)  # a valid export of the same handle, one second later
        got["rank1-differs"] = shard_import(lib, g, differs, 2.0)
        got["truncated"] = shard_import(lib, g, [blob[:-5]] * world, 2.0)
        got["config"] = shard_import(lib, g, [wrong] * world, 2.0)
        fresh_after += [is_fresh(d) for d in g]
        got["retry"] = shard_import(lib, g, [blob] * world, 2.0)
        want = {"not-fresh": _abi.STATE_NOT_FRESH, "rank1-differs": _abi.STATE_BAD_BLOB, "truncated": _abi.STATE_BAD_BLOB,
                "config": _abi.STATE_CONFIG_MISMATCH, "retry": _abi.STATE_OK}
        line["codes"] = got
        ok = all(got[k] == [v] * world for k, v in want.items()) and all(fresh_after)
        line["fresh_after_refusals"] = all(fresh_after)
        # the loaded group exports the single handle's bytes; the old entry points refuse sharded handles
        exports = shard_export(lib, g, 2.0)
        line["export_equal"] = all(e == blob for e in exports)
        ok = ok and line["export_equal"]
        line["old_calls_refuse"] = all(lib.yd_export_state(d._h, T.ns(2.0), None, 0) == 0 for d in g) and all(
            lib.yd_import_state(d._h, T.ns(2.0), blob, len(blob)) == _abi.STATE_UNSUPPORTED for d in dirty)
        ok = ok and line["old_calls_refuse"]
        try:
            src.import_state(blob, now=2.0)
        except StateError as e:
            line["single_refuses_not_fresh"] = e.code == _abi.STATE_NOT_FRESH
        d = fake_stats(world) - stats0
        line["same_collectives"] = bool((d == d[0]).all())
        ok = ok and line["same_collectives"]
    finally:
        for grp in groups:
            close_group(lib, grp)
        src.close()
        other.close()
    line["ok"] = bool(ok)
    print(json.dumps(line), flush=True)
    return ok


def summary(h, name, world, ok, **extra):
    c = dict(h.counts)
    for k in ("export_s", "import_s"):
        v = c.pop(k)
        c[k.replace("_s", "_ms_max")] = round(1e3 * max(v), 3) if v else None
        c[k.replace("_s", "_ms_median")] = round(1e3 * float(np.median(v)), 3) if v else None
    line = {"case": name, "world": world, "ok": ok, **c, **extra}
    print(json.dumps(line), flush=True)
    return line


def main():
    a = parse_args()
    ok = True
    targets = [int(x) for x in a.targets.split(",") if x]
    for k, s in enumerate(int(x) for x in a.fuzz.split(",") if x):
        h, good = fuzz_case(s, a.world, a.mode, targets, a.cuts, a.seed * 1000 + k)
        summary(h, f"fuzz-{s}", a.world, good, mode=a.mode)
        ok = ok and good
    for name in [x for x in a.scale.split(",") if x]:
        h, good = scale_case(name, a.world)
        summary(h, name, a.world, good, mode="handover")
        ok = ok and good
    if a.refusals:
        ok = refusal_case(a.world) and ok
    a4 = (C.c_ulonglong * 4)()
    T.FAKE.yd_fake_nccl_stats(0, a4)
    print(json.dumps({"shard_state": ok, "world": a.world, "fake_nccl_collectives": int(a4[0]),
                      "torch_loaded": "torch" in sys.modules}), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
