#!/usr/bin/env python
"""The packed solve of a range-sharded group (yd_shard_wait_for_starting_new_tasks_packed, include/ydshard.h) on ONE
GPU: W rank handles in W threads of one process, over the test-only NCCL stand-in, with tests/shard_threads_check.py's
harness (imported: it takes the same arguments, and loads the stand-in -- or, with --real-nccl, torch's libnccl.so.2 --
before anything else).

Every stream runs on two groups in lock-step, fed the same events with the same cut points and staging:
  packed group    most solves through the packed call (16-byte ranges up, 8-byte grants down), the rest through the
                  unpacked call; every packed solve is checked against ONE CPU checker handle fed the concatenated queue
                  through its own yd_wait_for_starting_new_tasks_packed: the ranks' grants, concatenated, equal the
                  checker's bit for bit, every rank's ids equal the checker's, and after every event the servant state,
                  next task id and lease counts equal the checker's (the harness's own checks)
  unpacked twin   every solve through the unpacked group call; its grants must equal the packed group's unpacked ones,
                  and the stand-in must record the same collectives (calls, all-gathers, all-reduces) for both
Cases:
  --fuzz SEEDS      seeded fuzz streams (zombies, servant expiry, frees of packed-granted and unknown ids, keep-alives,
                    heartbeats, ticks, several servants behind one IP: the whole-queue fallback)
  --config NAMES    shard_threads_check's CONFIGS, and here: lease (YD_LEASE_PREFETCH, leases near 0, near 30 000 ms and
                    2^31 - 1 ms, ticks 1 ms before and after each expiry), fallback (packed only, no twin: batches the
                    whole-queue fallback decides), many-classes (more than 256 classes: the fallback after the class
                    bound stops growing)
  --refusals        the packed call's refusals, each on every rank with no state change; the process must run with
                    YDSCHED_SHARD_PACKED_MAX_N (a lowered group-queue limit)

Prints one JSON line per case and a final {"shard_packed": ...} line; exit code 0 iff everything matched.
"""
import ctypes as C
import json
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import shard_threads_check as T  # noqa: E402  (parses the arguments, loads the NCCL the ranks use)

import numpy as np  # noqa: E402

from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT8_DTYPE, GRANT_DTYPE, PACKED_IDS_DTYPE, STATUS_GRANTED  # noqa: E402
from yadcc_b200.dispatcher import Servant, TaskDispatcher, pack_requests, unpack_grants  # noqa: E402

ARGS, FAKE, ns, par, Mismatch = T.ARGS, T.FAKE, T.ns, T.par, T.Mismatch


def sentinel_grants8(n: int) -> np.ndarray:
    g = np.zeros(max(n, 1), dtype=GRANT8_DTYPE)
    g.view(np.uint32)[:] = 0xDEADBEEF
    return g


class PackedHarness(T.Harness):
    """A group whose solves go through the packed call with probability p_packed (its own generator, so that the cut
    points and staging draws stay those of a twin with another p_packed)."""

    def __init__(self, name, world, seed, oracle=True, p_packed=0.75):
        super().__init__(name, world, seed, oracle)
        self.p_packed = p_packed
        self.mode_rng = np.random.default_rng(seed + 77)
        self.solves: list = []  # (packed, grants, collectives {calls, all-gathers, all-reduces} or None)
        self.marks: list = []  # the checker's lease count at each ("mark",) event
        self.counts.update(packed=0, unpacked=0, packed_staged_ranks=0, packed_handbacks=0, packed_granted=0)

    def solve(self, now, full):
        before = self.fake_stats()
        hb = self.counts["handbacks"]
        packed = bool(self.mode_rng.random() < self.p_packed)
        g = self.solve_packed(now, full) if packed else super().solve(now, full)
        self.counts["packed" if packed else "unpacked"] += 1
        if packed:
            self.counts["packed_handbacks"] += self.counts["handbacks"] - hb
            self.counts["packed_granted"] += int((g["status"] == STATUS_GRANTED).sum())
        d = None if before is None else [int(x) for x in (self.fake_stats() - before)[0][:3]]
        self.solves.append((packed, g, d))
        return g

    def solve_packed(self, now, full):
        # the same generator draws, in the same order, as shard_threads_check.Harness.solve
        W, n = self.W, len(full)
        cuts = self.cuts = self.cut_points(n)
        staged = self.rng.random(W) < 0.4
        full = np.ascontiguousarray(full)
        r16 = pack_requests(full)
        parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(W)]
        parts16 = [np.ascontiguousarray(r16[cuts[r]:cuts[r + 1]]) for r in range(W)]
        for r in range(W):
            if staged[r]:  # the 24-byte range, sometimes followed by unrelated requests
                q = parts[r]
                if self.rng.random() < 0.5 and n:
                    q = np.concatenate([q, full[: int(self.rng.integers(1, n + 1))]])
                self.ranks[r].stage_requests(np.ascontiguousarray(q))
                self.counts["packed_staged_ranks"] += 1
        outs = [sentinel_grants8(len(p)) for p in parts16]
        ids = [np.zeros(1, dtype=PACKED_IDS_DTYPE) for _ in range(W)]
        before = self.fake_stats()

        def call(r):
            p = parts16[r]
            return self.lib.yd_shard_wait_for_starting_new_tasks_packed(
                self.ranks[r]._h, ns(now), None if staged[r] else p.ctypes.data, len(p), outs[r].ctypes.data,
                ids[r].ctypes.data)
        rcs = par([lambda r=r: call(r) for r in range(W)])
        self.counts["solves"] += 1
        if any(rc != 0 for rc in rcs):
            self.fail("packed sharded solve did not decide the batch", rcs=rcs, staged=staged.tolist())
        mine = [(int(x["first_task_id"]), int(x["stride"])) for x in (i[0] for i in ids)]
        if any(m != mine[0] for m in mine):
            self.fail("ids differ between ranks", ids=mine)
        g8 = np.concatenate([outs[r][: len(parts16[r])] for r in range(W)])
        g = unpack_grants(g8, ids[0][0])
        if self.oracle is not None:
            o8, oids = self.oracle.wait_for_starting_new_tasks_packed(r16, now, unpack=False)
            want = (int(oids["first_task_id"]), int(oids["stride"]))
            if mine[0] != want:
                self.fail("ids differ from the checker's", sharded=mine[0], single=want)
            g1 = unpack_grants(o8, oids)
            bad = (g["status"] != g1["status"]) | (g["servant_index"] != g1["servant_index"]) | (g["task_id"] != g1["task_id"])
            bad |= (g8["servant_index"] != o8["servant_index"]) | (g8["status_ordinal"] != o8["status_ordinal"])
            if bad.any():
                i = int(np.nonzero(bad)[0][0])
                r = int(np.searchsorted(cuts, i, side="right") - 1)
                self.fail("packed grants differ", rank=r, index=i, local_index=i - cuts[r], mismatches=int(bad.sum()),
                          sharded=[int(x) for x in g8[i]], single=[int(x) for x in o8[i]], staged=staged.tolist())
        self.check_solve_stats(before)
        ok = g["status"] == STATUS_GRANTED
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        return g

    def event(self, ev, build):
        if ev[0] == "mark":
            if self.oracle is not None:
                self.marks.append(self.oracle.num_tasks())
            return
        super().event(ev, build)


def builder(streams, handles, k):
    """The value of event k's per-handle request builder, checked equal on every handle (intern ids agree)."""
    def build(f):
        vals = [streams[h].events[k][2](handles[h]) for h in range(len(handles))]
        for v in vals[1:]:
            assert v.shape == vals[0].shape and (v == vals[0]).all(), "intern ids differ between handles"
        return vals[0]
    return build


def run_pair(name, world, make, seed, p_packed=0.75, twin=True):
    """`make(handle)` -> Stream, run on the packed group (checked against the checker) and, in lock-step, on the
    unpacked twin."""
    h = PackedHarness(name, world, seed, True, p_packed)
    t = PackedHarness(name + "/unpacked", world, seed, False, 0.0) if twin else None
    ok = True
    try:
        hh = h.ranks + [h.oracle]
        streams = [make(d) for d in hh]
        tstreams = [make(d) for d in t.ranks] if t else []
        base = streams[-1]
        for k, ev in enumerate(base.events):
            for other in streams[:-1] + tstreams:
                e2 = other.events[k]
                if ev[0] in ("wait", "enqueue") and not callable(e2[-1]):
                    assert ev[-1].shape == e2[-1].shape and (ev[-1] == e2[-1]).all(), "intern ids differ between handles"
            h.event(ev, builder(streams, hh, k))
            if t is None:
                continue
            t.event(tstreams[0].events[k], builder(tstreams, t.ranks, k))
            if len(h.solves) != len(t.solves):
                h.fail("the twin made a different number of solves")
            if h.solves and len(h.solves) > h.counts.get("twin_checked", 0):
                h.counts["twin_checked"] = len(h.solves)
                (packed, g, d), (_, g2, d2) = h.solves[-1], t.solves[-1]
                if len(g) != len(g2) or any((g[f] != g2[f]).any() for f in ("status", "servant_index", "task_id")):
                    h.fail("packed and unpacked group calls decided differently", packed=packed)
                if d != d2:
                    h.fail("packed and unpacked group calls made different collectives", packed=d, unpacked=d2)
                h.counts["twin_equal_packed"] = h.counts.get("twin_equal_packed", 0) + int(packed)
    except Mismatch:
        ok = False
    line = {"case": name, "world": world, "ok": ok, "twin": t is not None}
    line.update(h.counts)
    if h.marks:
        line["marks"] = h.marks
    print(json.dumps(line), flush=True)
    h.close()
    if t:
        t.close()
    return line


# ---- streams ------------------------------------------------------------------------------------------------------------
LEASES_MS = [0, 1, 2, 29_999, 30_000, 30_001, (1 << 31) - 1]


def lease_stream(d: TaskDispatcher) -> S.Stream:
    """cfg2-mod-small's cluster, servants alive for 35 days; one batch whose leases cycle through LEASES_MS, half of them
    prefetches; then for every lease length L > 0 a tick 1 ms before its expiry and one 1 ms after, each followed by a
    heartbeat of every servant (the first tick keeps the leases, the second makes zombies of them, which the heartbeats
    sweep)."""
    w = S.config2(5000, 200, 8, variant="mod")
    ev: list = [("hb", 0.0, sv, 3.0e6) for sv in w.servants]
    r = w.build_requests(d)
    r["expires_in_ns"] = np.asarray(LEASES_MS, dtype=np.int64)[np.arange(len(r)) % len(LEASES_MS)] * 1_000_000
    r["flags"] = np.where(np.random.default_rng(4).random(len(r)) < 0.5, _abi.REQ_FLAG_PREFETCH, 0).astype(r["flags"].dtype)
    t0 = 1.0
    ev.append(("wait", t0, r))
    # a tick turns the expired leases into zombies; every servant's heartbeat then sweeps them ("mark": the checker's
    # lease count)
    sweep = [("notify", sv.observed_location, []) for sv in w.servants] + [("mark",)]
    for L in LEASES_MS[1:]:
        ev += [("tick", t0 + (L - 1) / 1000)] + sweep + [("tick", t0 + (L + 1) / 1000)] + sweep
    return S.Stream("lease", ev)


def many_classes_workload() -> S.Workload:
    """cfg2-mod's servants, min_version 0..39 over 8 digests: 320 classes, more than the class bound can grow to."""
    w = S.config2(4000, 160, 8, variant="mod")
    inner = w.build_requests

    def build(d):
        r = inner(d)
        r["min_version"] = np.random.default_rng(6).integers(0, 40, len(r)).astype(np.uint32)
        return r
    return S.Workload("many-classes", w.servants, w.digests, build)


def fuzz(seed):
    return lambda d: S.fuzz_stream(d, seed, n_servants=8 + seed % 30, unique_hosts=ARGS.unique_hosts)


# ---- refusals -----------------------------------------------------------------------------------------------------------
def refusal_case(world):
    """Each refusal returns 1 on every rank, writes no grant and changes no state (next task id, servant state, lease
    counts compared before and after): a handle not in a group, n_local above the staged count, a wide cluster, and a
    group queue above the packed limit made of ranges that each stay below it (given, and staged: the staged queues
    survive the refusal)."""
    limit = int(os.environ["YDSCHED_SHARD_PACKED_MAX_N"])
    h = PackedHarness("packed-refusals", world, 3, oracle=True, p_packed=1.0)
    line = {"case": "packed-refusals", "world": world, "limit": limit}
    ok = True

    def snapshot():
        return ([d.next_task_id() for d in h.ranks], [d.servant_state().copy() for d in h.ranks],
                [d.num_tasks() for d in h.ranks])

    def unchanged(before, what):
        after = snapshot()
        for r in range(world):
            if after[0][r] != before[0][r] or after[2][r] != before[2][r] or \
                    any((after[1][r][f] != before[1][r][f]).any() for f in after[1][r].dtype.names):
                h.fail(f"{what}: a refused call changed the state", rank=r)

    def packed_call(reqs16, n, staged=False):
        outs = [sentinel_grants8(n[r]) for r in range(world)]
        ids = [np.zeros(1, dtype=PACKED_IDS_DTYPE) for _ in range(world)]
        before = h.fake_stats()
        rcs = par([lambda r=r: h.lib.yd_shard_wait_for_starting_new_tasks_packed(
            h.ranks[r]._h, ns(1.0), None if staged else reqs16[r].ctypes.data, n[r], outs[r].ctypes.data,
            ids[r].ctypes.data) for r in range(world)])
        d = None if before is None else (h.fake_stats() - before)
        return rcs, outs, d

    try:
        w = S.config2(5000, 200, 8, variant="mod")
        h.every(lambda d: [d.keep_servant_alive(sv, 100.0, now=0.0) for sv in w.servants])
        fulls = [w.build_requests(d) for d in h.ranks + [h.oracle]]
        full = fulls[-1]
        r16 = pack_requests(full)

        # 1. a handle that has not joined a group
        lone = TaskDispatcher(h.lib)
        lone.keep_servant_alive(w.servants[0], 100.0, now=0.0)
        n0, s0 = lone.next_task_id(), lone.servant_state().copy()
        o = sentinel_grants8(4)
        rc = h.lib.yd_shard_wait_for_starting_new_tasks_packed(lone._h, ns(1.0), r16.ctypes.data, 4, o.ctypes.data, None)
        if rc != 1 or lone.next_task_id() != n0 or (lone.servant_state() != s0).any() or lone.num_tasks() != 0:
            h.fail("a handle outside a group was not refused", rc=rc)
        if (o.view(np.uint32) != 0xDEADBEEF).any():
            h.fail("a refused call wrote grants")
        lone.close()
        line["not_in_group"] = True

        # 2. n_local above the staged count (no collective)
        for r, d in enumerate(h.ranks):
            d.stage_requests(np.ascontiguousarray(fulls[r][:2]))
        before = snapshot()
        rcs, outs, d = packed_call(None, [3] * world, staged=True)
        if rcs != [1] * world or (d is not None and d.any()):
            h.fail("a staged packed solve longer than the staged queue was not refused before any exchange", rcs=rcs)
        unchanged(before, "staged count")
        line["staged_count"] = True

        # 3. the group queue above the limit: ranges that each stay below it, summing to limit + 1 (and to the limit:
        # decided, so the rule is on the sum).  Staged, the refusal keeps the staged queues, which the unpacked group call
        # then decides as the checker decides them.
        if world >= 2:
            sizes = [limit // world + (1 if r < limit % world else 0) for r in range(world)]
            assert sum(sizes) == limit and max(sizes) < limit
            over = list(sizes)
            over[-1] += 1
            assert max(over) <= limit
            cut = np.concatenate([[0], np.cumsum(over)])
            assert cut[-1] <= len(full)
            parts16 = [np.ascontiguousarray(r16[cut[r]:cut[r + 1]]) for r in range(world)]
            staged = [np.ascontiguousarray(fulls[r][cut[r]:cut[r + 1]]) for r in range(world)]
            before = snapshot()
            rcs, outs, d = packed_call(parts16, over)
            if rcs != [1] * world:
                h.fail("a group queue above the packed limit was not refused", rcs=rcs, sizes=over)
            if any((o.view(np.uint32) != 0xDEADBEEF).any() for o in outs):
                h.fail("a refused call wrote grants")
            # the lengths travel with exchange 1: one all-gather, nothing after it
            if d is not None and not ((d[:, 0] == 1) & (d[:, 1] == 1) & (d[:, 2] == 0)).all():
                h.fail("the refusal was not decided at the first exchange", calls=d.tolist())
            unchanged(before, "group queue")
            # (an upload empties the staging area, as in the unpacked call: the staged form is refused with the staged
            # queues kept)
            for r, dd in enumerate(h.ranks):
                dd.stage_requests(staged[r])
            rcs, outs, d = packed_call(None, over, staged=True)
            if rcs != [1] * world:
                h.fail("a staged group queue above the packed limit was not refused", rcs=rcs)
            unchanged(before, "staged group queue")
            # the unpacked call's limit is not the packed one: the same staged ranges are decided
            gouts = [np.zeros(max(k, 1), dtype=GRANT_DTYPE) for k in over]
            rcs = par([lambda r=r: h.lib.yd_shard_wait_for_starting_new_tasks(h.ranks[r]._h, ns(1.0), None, over[r],
                                                                              gouts[r].ctypes.data) for r in range(world)])
            if rcs != [0] * world:
                h.fail("the unpacked call refused the staged ranges", rcs=rcs)
            g = np.concatenate([gouts[r][:over[r]] for r in range(world)])
            g1 = h.oracle.wait_for_starting_new_tasks(np.ascontiguousarray(full[: cut[-1]]), 1.0)
            if any((g[f] != g1[f]).any() for f in ("status", "servant_index", "task_id")):
                h.fail("the staged ranges kept through the refusal were not decided as the checker decides them")
            h.ev = ("state",)
            h.compare(True)
            # exactly the limit: decided, equal to the checker
            cut = np.concatenate([[0], np.cumsum(sizes)])
            parts16 = [np.ascontiguousarray(r16[cut[r]:cut[r + 1]]) for r in range(world)]
            rcs, outs, d = packed_call(parts16, sizes)
            if rcs != [0] * world:
                h.fail("a group queue of exactly the packed limit was refused", rcs=rcs, sizes=sizes)
            o8, oids = h.oracle.wait_for_starting_new_tasks_packed(np.ascontiguousarray(r16[: cut[-1]]), 1.0, unpack=False)
            g8 = np.concatenate([outs[r][: sizes[r]] for r in range(world)])
            if (g8.view(np.uint32) != o8.view(np.uint32)).any():
                h.fail("a group queue of exactly the packed limit was decided differently from the checker")
            h.compare(True)
            line["group_limit"] = True

        # 4. a wide cluster (capacities above 8192 per servant): no collective
        wide = Servant("10.9.0.1:8000", None, [w.digests[0]], 8, 40000, 0, 64 << 30, 40 << 30, 70000, _abi.PRIORITY_USER)
        h.every(lambda d: d.keep_servant_alive(wide, 100.0, now=0.5))
        before = snapshot()
        n = [min(len(r16), 4)] * world
        rcs, outs, d = packed_call([np.ascontiguousarray(r16[:4])] * world, n)
        if rcs != [1] * world or (d is not None and d.any()):
            h.fail("a wide cluster was not refused before any exchange", rcs=rcs)
        unchanged(before, "wide")
        line["wide"] = True
    except Mismatch:
        ok = False
    line["ok"] = ok
    print(json.dumps(line), flush=True)
    h.close()
    return ok


def main():
    a = ARGS
    ok = True
    k = 0
    for s in [int(x) for x in a.fuzz.split(",") if x]:
        line = run_pair(f"fuzz-{s}" + ("-unique" if a.unique_hosts else ""), a.world, fuzz(s), a.seed * 1000 + k)
        ok = ok and line["ok"]
        k += 1
    for c in [x for x in a.config.split(",") if x]:
        if c == "lease":
            line = run_pair(c, a.world, lease_stream, a.seed * 1000 + k, p_packed=1.0)
            tt = line.get("marks", [])
            # every tick before an expiry keeps the leases, every tick after one makes zombies of some
            swept = len(tt) == 2 * (len(LEASES_MS) - 1) and all(tt[i] > tt[i + 1] for i in range(0, len(tt), 2))
            if not swept:
                print(json.dumps({"case": c, "error": "the ticks did not straddle every expiry", "marks": tt}))
            ok = ok and line["ok"] and swept
        elif c == "fallback":
            line = run_pair(c, a.world, fuzz(3), a.seed * 1000 + k, p_packed=1.0, twin=False)
            ok = ok and line["ok"]
        else:
            make = many_classes_workload if c == "many-classes" else T.CONFIGS[c]
            line = run_pair(c, a.world, lambda d, make=make: T.workload_stream(make(), d), a.seed * 1000 + k)
            ok = ok and line["ok"]
        k += 1
    if a.refusals:
        ok = refusal_case(a.world) and ok
    final = {"shard_packed": ok, "world": a.world, "nccl": "real" if FAKE is None else "fake_nccl"}
    if FAKE is not None:
        a4 = (C.c_ulonglong * 4)()
        FAKE.yd_fake_nccl_stats(0, a4)
        final["fake_nccl_collectives"] = int(a4[0])
        final["torch_loaded"] = "torch" in sys.modules
    print(json.dumps(final), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
