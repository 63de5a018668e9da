#!/usr/bin/env python
"""The pre-filtered solve of a range-sharded group (yd_shard_filter_and_wait_for_starting_new_tasks and
yd_shard_derive_filter_and_wait_for_starting_new_tasks, include/ydshard.h) on ONE GPU: W rank handles in W threads of
one process, over the test-only NCCL stand-in (tests/fake_nccl/libnccl.so.2, loaded with RTLD_GLOBAL before anything
else; this process must not import torch).  With --real-nccl the process imports torch first and runs over the real
NCCL.

Every call is checked exactly against ONE CPU checker handle (checkers/libydport_keys.so, which has both single-handle
calls) fed the concatenated queue -- for descriptors, the ranks' argument tables appended in rank order: every rank's
verdicts, hits, returned count and grants; after every call every servant's running_tasks and every replica's next task
id.  Each call is followed by the staged offered queue decided again, a plain sharded solve and a collective free.
  --fuzz N    N seeded calls per stage set (none, cache, dedupe, both) and per kind (keys, descriptors), random cuts
              (empty ranges included), a range filtered out entirely, everything filtered out, a refusal of one rank's
              descriptors, and batches with requestors behind servant IPs (the sequential fallback)
  --config3   the configs[3] descriptor queue (streams.config3_task_sources, 100 k) over cfg2-mod's servants

Prints one JSON line per case and a final {"shard_filter": ...} line; exit code 0 iff everything matched.
"""
import argparse
import ctypes as C
import json
import sys
import threading
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE_NCCL = ROOT / "tests" / "fake_nccl" / "libnccl.so.2"
CHECKER = ROOT / "checkers" / "libydport_keys.so"

ap = argparse.ArgumentParser()
ap.add_argument("--world", type=int, default=2)
ap.add_argument("--fuzz", type=int, default=0, help="calls per (stage set, kind)")
ap.add_argument("--config3", action="store_true")
ap.add_argument("--real-nccl", action="store_true")
ap.add_argument("--seed", type=int, default=0)
ARGS = ap.parse_args()
if ARGS.real_nccl:
    import torch  # noqa: F401  (its libnccl.so.2 is the one the scheduler's dlopen finds)
    FAKE = None
else:
    FAKE = C.CDLL(str(FAKE_NCCL), mode=C.RTLD_GLOBAL)

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import FILTER_CACHE_HIT, FILTER_JOINED, FILTER_OFFERED, GRANT_DTYPE, REQ_DTYPE, STATUS_GRANTED  # noqa: E402
from yadcc_b200.dispatcher import RunningTask, Servant, TaskDispatcher, TaskSources  # noqa: E402

if FAKE is not None:
    assert "torch" not in sys.modules, "torch loads the real libnccl.so.2"

REFUSED = (1 << 64) - 1


def ns(now: float) -> int:
    return int(round(now * 1_000_000_000))


def par(fns):
    """Run fns in one thread each (ctypes releases the GIL); return their results in order."""
    out, err = [None] * len(fns), []

    def run(i, f):
        try:
            out[i] = f()
        except BaseException as e:  # noqa: BLE001
            err.append(e)

    ts = [threading.Thread(target=run, args=(i, f)) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if err:
        raise err[0]
    return out


class Mismatch(Exception):
    pass


def hexrows(rng, n):
    b = np.frombuffer(rng.bytes(32 * n), dtype=np.uint8).reshape(n, 32)
    h = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    return np.ascontiguousarray(np.stack([h[b >> 4], h[b & 15]], axis=2).reshape(n, 64))


class Group:
    """W rank handles joined to one group, and the checker fed the concatenated queue."""

    def __init__(self, name: str, world: int, seed: int):
        self.name, self.W = name, world
        self.rng = np.random.default_rng(seed)
        self.lib = _abi.load_library()
        self.ranks = [TaskDispatcher(self.lib) for _ in range(world)]
        self.oracle = TaskDispatcher(str(CHECKER))
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        assert self.lib.yd_shard_unique_id(uid) == 0, "yd_shard_unique_id"
        rcs = par([lambda r=r: self.lib.yd_shard_init(self.ranks[r]._h, r, world, uid) for r in range(world)])
        assert rcs == [0] * world, f"yd_shard_init: {rcs}"
        self.counts = {"calls": 0, "offered": 0, "cache_hits": 0, "joined": 0, "joined_across": 0, "empty_ranges": 0,
                       "filtered_ranges": 0, "all_filtered": 0, "handbacks": 0, "refusals": 0, "redecided": 0}
        self.outstanding: dict[int, int] = {}
        self.holder: dict[int, int] = {}  # task id -> rank whose range held the request
        self.ev = None

    @property
    def handles(self):
        return self.ranks + [self.oracle]

    def close(self):
        for d in self.ranks:
            self.lib.yd_shard_finalize(d._h)
            d.close()
        self.oracle.close()

    def fail(self, what: str, **kw):
        line = {"case": self.name, "world": self.W, "event": self.ev, "error": what}
        line.update(kw)
        print(json.dumps(line, default=str), flush=True)
        raise Mismatch(what)

    def fake_gathers(self):
        if FAKE is None:
            return None
        a = (C.c_ulonglong * 4)()
        FAKE.yd_fake_nccl_stats(0, a)
        return int(a[1])

    def cut(self, n, cuts=None):
        if cuts is None:
            cuts = sorted([0, n] + [int(x) for x in self.rng.integers(0, n + 1, self.W - 1)])
        return cuts

    def compare(self):
        ref = self.oracle.servant_state()
        for r, d in enumerate(self.ranks):
            st = d.servant_state()
            if len(st) != len(ref) or (st["running_tasks"] != ref["running_tasks"]).any():
                self.fail("running_tasks differ", rank=r)
            if d.next_task_id() != self.oracle.next_task_id():
                self.fail("next_task_id differs", rank=r, group=d.next_task_id(), single=self.oracle.next_task_id())

    def record(self, grants, ranks_of):
        ok = grants["status"] == STATUS_GRANTED
        for tid, sidx, r in zip(grants["task_id"][ok].tolist(), grants["servant_index"][ok].tolist(), ranks_of[ok].tolist()):
            self.outstanding[tid] = sidx
            self.holder[tid] = r

    # -- the calls -----------------------------------------------------------------------------------------------------
    def solve(self, now, full, cuts=None):
        """A plain sharded solve of host ranges, checked against the checker."""
        cuts = self.cut(len(full), cuts)
        parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(self.W)]
        outs = [np.zeros(max(len(p), 1), dtype=GRANT_DTYPE) for p in parts]
        rcs = par([lambda r=r: self.lib.yd_shard_wait_for_starting_new_tasks(
            self.ranks[r]._h, ns(now), parts[r].ctypes.data, len(parts[r]), outs[r].ctypes.data) for r in range(self.W)])
        if any(rcs):
            self.fail("sharded solve refused", rcs=rcs)
        g = np.concatenate([outs[r][:len(parts[r])] for r in range(self.W)])
        g1 = self.oracle.wait_for_starting_new_tasks(np.ascontiguousarray(full), now).copy()
        if g.tolist() != g1.tolist():
            self.fail("plain solve grants differ")
        self.record(g, np.repeat(np.arange(self.W), np.diff(cuts)))
        self.compare()
        return g

    def free(self, frac=0.5):
        """A collective free of a seeded `frac` of the outstanding leases, the ids passed on the last rank."""
        if not self.outstanding:
            return
        ids = np.asarray(sorted(self.outstanding), dtype=np.uint64)
        ids = np.ascontiguousarray(ids[self.rng.random(len(ids)) < frac])
        empty = np.zeros(0, dtype=np.uint64)
        args = [ids if r == self.W - 1 else empty for r in range(self.W)]
        rcs = par([lambda r=r: self.lib.yd_shard_free_tasks(self.ranks[r]._h, args[r].ctypes.data if len(args[r]) else None,
                                                             len(args[r])) for r in range(self.W)])
        if any(rcs):
            self.fail("yd_shard_free_tasks failed", rcs=rcs)
        self.oracle.free_tasks(ids)
        for i in ids.tolist():
            self.outstanding.pop(i, None)
        self.compare()

    def filtered(self, now, full, cuts, *, keys=None, digests=None, srcs=None, stages=0, refuse=False):
        """One group pre-filtered call (keys: `keys` / `digests` of the whole queue; descriptors: srcs[r] per rank),
        checked against the checker's single-handle call on the concatenated queue.  Returns each rank's offered count."""
        W = self.W
        parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(W)]
        counts = [len(p) for p in parts]
        g0 = self.fake_gathers()
        if srcs is None:
            sl = lambda m, r: None if m is None else np.ascontiguousarray(m[cuts[r]:cuts[r + 1]])  # noqa: E731
            got = par([lambda r=r: self.ranks[r]._filter_with(self.lib.yd_shard_filter_and_wait_for_starting_new_tasks,
                                                              parts[r], sl(keys, r), sl(digests, r), now, None, None, True)
                       for r in range(W)])
            want = self.oracle.filter_and_wait_for_starting_new_tasks(np.ascontiguousarray(full), keys, digests, now)
        else:
            def raw(r):  # the C call itself: the return value on every rank is part of the contract
                v = np.zeros(counts[r], dtype=np.uint8)
                h = np.zeros(counts[r], dtype=_abi.RUNNING_HIT_DTYPE)
                o = np.zeros(max(counts[r], 1), dtype=GRANT_DTYPE)
                f = srcs[r].struct()
                k = self.lib.yd_shard_derive_filter_and_wait_for_starting_new_tasks(
                    self.ranks[r]._h, ns(now), parts[r].ctypes.data, counts[r], C.byref(f), stages, v.ctypes.data,
                    h.ctypes.data, o.ctypes.data)
                return (v, h, o[:k]) if k != REFUSED else None
            got = par([lambda r=r: raw(r) for r in range(W)])
            if refuse:
                if any(x is not None for x in got):
                    self.fail("a refused descriptor queue was not refused on every rank",
                              refused=[x is None for x in got])
                if self.oracle.next_task_id() != self.ranks[0].next_task_id():
                    self.fail("next_task_id differs after a refusal")
                self.counts["refusals"] += 1
                self.compare()
                return None
            want = self.oracle.derive_filter_and_wait_for_starting_new_tasks(
                np.ascontiguousarray(full), TaskSources.concat(srcs, counts), stages, now)
        if any(x is None for x in got):
            self.fail("the call was refused", refused=[x is None for x in got])
        v1, h1, g1 = want
        lo, first, offered = 0, 0, []
        for r in range(W):
            v, h, g = got[r]
            hi = lo + counts[r]
            mine = int((v1[lo:hi] == FILTER_OFFERED).sum())
            if v.tolist() != v1[lo:hi].tolist():
                self.fail("verdicts differ", rank=r)
            if h.tolist() != h1[lo:hi].tolist():
                self.fail("hits differ", rank=r)
            if len(g) != mine:
                self.fail("offered counts differ", rank=r, group=len(g), single=mine)
            if g.tolist() != g1[first:first + mine].tolist():
                self.fail("grants differ", rank=r)
            for j in np.nonzero(v == FILTER_JOINED)[0].tolist():
                e = self.oracle.running_index_entry(int(h["snapshot_index"][j]))
                self.counts["joined_across"] += int(self.holder.get(e.task_grant_id, r) != r)
            self.counts["empty_ranges"] += int(counts[r] == 0)
            self.counts["filtered_ranges"] += int(counts[r] > 0 and mine == 0)
            offered.append(mine)
            lo, first = hi, first + mine
        self.counts["all_filtered"] += int(len(full) > 0 and sum(offered) == 0)
        self.counts["calls"] += 1
        self.counts["offered"] += sum(offered)
        self.counts["cache_hits"] += int((v1 == FILTER_CACHE_HIT).sum())
        self.counts["joined"] += int((v1 == FILTER_JOINED).sum())
        if g0 is not None:
            gathers = self.fake_gathers() - g0 - (1 if srcs is not None else 0)  # (the descriptors' agreement)
            self.counts["handbacks"] += gathers % 2  # the ranges' all-gather of a batch the sequential solver decided
        offered_ranks = np.repeat(np.arange(W), offered)
        self.record(g1, offered_ranks)
        # every rank's stats report its own stages
        for r in range(W):
            st = self.ranks[r].last_solve_stats()
            if st is None or st["decisions"] != counts[r] or (counts[r] and st["prep_ms"] <= 0):
                self.fail("last_solve_stats does not report the call", rank=r, stats=st)
        self.compare()
        return offered

    def redecide(self, now, offered):
        """The offered requests stay staged: yd_shard_wait_for_starting_new_tasks(NULL, offered) decides them again."""
        outs = [np.zeros(max(k, 1), dtype=GRANT_DTYPE) for k in offered]
        rcs = par([lambda r=r: self.lib.yd_shard_wait_for_starting_new_tasks(self.ranks[r]._h, ns(now), None, offered[r],
                                                                              outs[r].ctypes.data) for r in range(self.W)])
        if any(rcs):
            self.fail("deciding the staged offered requests was refused", rcs=rcs)
        g = np.concatenate([outs[r][:offered[r]] for r in range(self.W)])
        g1 = self.oracle.wait_for_staged_tasks(sum(offered), now) if sum(offered) else np.zeros(0, GRANT_DTYPE)
        if g.tolist() != g1.tolist():
            self.fail("the staged offered queue decided differently")
        self.record(g, np.repeat(np.arange(self.W), offered))
        self.counts["redecided"] += 1
        self.compare()


# ---- a small cluster, a bloom filter and an in-flight index --------------------------------------------------------------
DIGESTS = [f"{i:02x}" * 32 for i in range(4)]
N_TU, N_ARGS = 300, 14


def servants(rng):
    out = []
    for i in range(24):
        host = f"10.3.0.{i % 16}"  # 8 hosts with two servants: a requestor there needs the sequential solver
        envs = [DIGESTS[i % 4]] + ([DIGESTS[(i + 1) % 4]] if i == 5 else [])
        out.append(Servant(f"{host}:{8000 + i}", None, envs, 8, 8, int(rng.integers(0, 3)), 64 << 30, 48 << 30,
                           int(rng.choice([2, 4, 8])), _abi.PRIORITY_USER if i % 3 else _abi.PRIORITY_DEDICATED))
    return out


class Workload:
    """Requests are (TU, compiler) combinations: a TU has an argument string and a source digest."""

    def __init__(self, g: Group):
        rng = np.random.default_rng(7)
        self.g = g
        self.args = [bytes(rng.integers(32, 127, int(m), dtype=np.uint8)) for m in np.geomspace(40, 3000, N_ARGS).astype(int)]
        self.tu_args = rng.integers(0, N_ARGS, N_TU)
        self.tu_src = hexrows(rng, N_TU)
        self.env = [np.asarray([d.intern_env(x) for x in DIGESTS], dtype=np.uint32) for d in g.handles]
        self.outside = [np.asarray([d.intern_ip(f"172.20.0.{i}") for i in range(9)], dtype=np.uint32) for d in g.handles]
        self.inside = [np.asarray([d.intern_ip(f"10.3.0.{i}") for i in range(8)], dtype=np.uint32) for d in g.handles]
        assert all((e == self.env[-1]).all() for e in self.env), "intern ids differ between handles"
        self.cached: set = set()  # combos whose cache keys are in the bloom filter

    def queue(self, combos, inside_frac=0.0):
        g, rng = self.g, self.g.rng
        n = len(combos)
        r = np.zeros(n, dtype=REQ_DTYPE)
        r["env_id"] = self.env[-1][[c[1] for c in combos]] if n else 0
        r["min_version"] = rng.integers(0, 2, n)
        ips = np.where(rng.random(n) < inside_frac, self.inside[-1][rng.integers(0, 8, n)], self.outside[-1][rng.integers(0, 9, n)])
        r["requestor_ip"] = ips
        r["expires_in_ns"] = 10_000_000_000
        return r

    def combos(self, n, pool=None):
        rng = self.g.rng
        if pool is not None:
            pool = sorted(pool)
            return [pool[int(i)] for i in rng.integers(0, len(pool), n)]
        return [(int(t), int(e)) for t, e in zip(rng.integers(0, N_TU, n), rng.integers(0, 4, n))]

    def sources(self, combos, cuts):
        """Per rank its own argument table: the strings its range uses, in a shuffled order, plus an unused one."""
        out = []
        rng = self.g.rng
        for r in range(self.g.W):
            mine = combos[cuts[r]:cuts[r + 1]]
            used = sorted({int(self.tu_args[t]) for t, _ in mine} | {int(rng.integers(0, N_ARGS))})
            rng.shuffle(used)
            pos = {a: k for k, a in enumerate(used)}
            idx = np.asarray([pos[int(self.tu_args[t])] for t, _ in mine], dtype=np.uint32)
            sd = self.tu_src[[t for t, _ in mine]] if mine else self.tu_src[:0]
            out.append(TaskSources.of([self.args[a] for a in used], idx, sd))
        return out

    def keys(self, combos):
        """The cache keys and task digests of the combos, derived by the checker."""
        reqs = self.queue(combos)
        src = TaskSources.of(self.args, self.tu_args[[t for t, _ in combos]], self.tu_src[[t for t, _ in combos]])
        return self.g.oracle.derive_task_keys(reqs, src)


def index_from(g: Group, dm, grants):
    """Heartbeats reporting every granted request of `grants` as running, with its task digest (dm[j]); then the group's
    index refresh on every rank."""
    by: dict[int, list] = {}
    for j, gr in enumerate(grants.tolist()):
        tid, sidx, status = gr[0], gr[1], gr[2]
        if status == STATUS_GRANTED:
            by.setdefault(sidx, []).append(RunningTask(1000 + j, tid, g.oracle.servant_location(sidx), bytes(dm[j]).decode()))
    batch = [(g.oracle.servant_location(k), v) for k, v in sorted(by.items())]
    got = par([lambda d=d: d._notify_with(g.lib.yd_shard_notify_servants_running_tasks, batch) for d in g.ranks])
    want = g.oracle.notify_servants_running_tasks(batch)
    if any(x != want for x in got):
        g.fail("heartbeat answers differ")
    n = par([lambda d=d: int(g.lib.yd_shard_running_index_refresh(d._h)) for d in g.ranks])
    if any(x != g.oracle.running_index_refresh() for x in n):
        g.fail("index sizes differ")
    g.compare()


def run_fuzz(world: int, calls: int, case_seed: int) -> bool:
    g = Group("fuzz", world, case_seed)
    w = Workload(g)
    ok = True
    try:
        for sv in servants(np.random.default_rng(3)):
            for d in g.handles:
                d.keep_servant_alive(sv, 3600.0, now=0.0)
        rng = g.rng
        combos = sorted({(int(t), int(e)) for t, e in zip(rng.integers(0, N_TU, 600), rng.integers(0, 4, 600))})
        km, _ = w.keys(combos)
        for d in g.handles:
            d.bloom_reset(1 << 16, 4)
            d.bloom_add(km[0::3])
        w.cached = set(combos[0::3])
        # running combos: their leases are reported by heartbeats with their digests, the group's in-flight index
        running = combos[1::3]
        now = 1.0
        for kind in ("keys", "descriptors"):
            for stages in (0, 1, 2, 3):
                for k in range(calls):
                    now += 0.25
                    g.ev = f"{kind} stages {stages} call {k}"
                    if k % 5 == 0:  # fresh leases reported for running combos, and the index refreshed on every rank
                        sub = [running[int(i)] for i in rng.integers(0, len(running), 60)]
                        gr = g.solve(now, w.queue(sub))
                        index_from(g, w.keys(sub)[1], gr)
                        now += 0.05
                    n = int(rng.choice([0, 1, 3, 40, 150, 400]))
                    special = k % 7
                    pool = None
                    if special == 1 and stages & 1:
                        pool = w.cached  # everything filtered out
                    cs = w.combos(n, pool)
                    cuts = g.cut(n)
                    if special == 2:
                        cuts = sorted([0, 0] + cuts[1:])[:world + 1] if world > 1 else cuts  # rank 0's range empty
                        cuts[-1] = n
                    if special == 3 and stages & 1 and world > 1 and n:
                        # the last rank's range made of cached combos only: filtered out entirely
                        lo = cuts[-2]
                        cached = sorted(w.cached)
                        for j in range(lo, n):
                            cs[j] = cached[int(rng.integers(0, len(cached)))]
                    inside = 0.3 if special == 4 else 0.0  # requestors behind servant IPs: the sequential fallback
                    q = w.queue(cs, inside)
                    if kind == "keys":
                        km, dm = w.keys(cs) if n else (np.zeros((0, 81), np.uint8), np.zeros((0, 64), np.uint8))
                        offered = g.filtered(now, q, cuts, keys=km if stages & 1 else None,
                                             digests=dm if stages & 2 else None)
                    else:
                        srcs = w.sources(cs, cuts)
                        offered = g.filtered(now, q, cuts, srcs=srcs, stages=stages)
                        if special == 5 and n:
                            # one rank's descriptors refused: every rank refuses, and the staged queues are kept
                            bad = [TaskSources(s.args, s.args_offsets, s.args_index.copy(), s.source_digests) for s in srcs]
                            rr = int(rng.integers(0, world))
                            while cuts[rr + 1] == cuts[rr]:
                                rr = (rr + 1) % world
                            bad[rr].args_index[-1] = len(bad[rr].args_offsets) - 1
                            g.ev += " refusal"
                            g.filtered(now + 0.01, q, cuts, srcs=bad, stages=stages, refuse=True)
                    g.redecide(now + 0.02, offered)
                    g.solve(now + 0.03, w.queue(w.combos(int(rng.integers(0, 30)))))
                    g.free()
    except Mismatch:
        ok = False
    print(json.dumps({"case": "fuzz", "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    return ok


def run_config3(world: int, case_seed: int) -> bool:
    """The configs[3] descriptor queue (100 k) over cfg2-mod's servants: cut into W ranges, each with the whole argument
    table, so the checker's concatenated table holds W copies; stages both, after an index from a first call's grants."""
    g = Group("config3", world, case_seed)
    ok = True
    try:
        wl = S.config2(100_000, 2000, 8, seed=42, variant="mod")
        for d in g.handles:
            wl.register(d)
        reqs = [wl.build_requests(d) for d in g.handles]
        assert all((r == reqs[-1]).all() for r in reqs), "intern ids differ between handles"
        q = np.ascontiguousarray(reqs[-1])
        src = S.config3_task_sources(100_000)
        n = len(q)
        cuts = [n * r // world for r in range(world + 1)]
        srcs = [TaskSources(src.args, src.args_offsets, np.ascontiguousarray(src.args_index[cuts[r]:cuts[r + 1]]),
                            np.ascontiguousarray(src.source_digests[cuts[r]:cuts[r + 1]])) for r in range(world)]
        km, dm = g.oracle.derive_task_keys(q[:20_000].copy(), TaskSources(src.args, src.args_offsets, src.args_index[:20_000],
                                                                          src.source_digests[:20_000]))
        for d in g.handles:
            d.bloom_reset(27584639, 10)
            d.bloom_add(km[::4])
        g.ev = "config3 first call"
        offered = g.filtered(1.0, q, cuts, srcs=srcs, stages=_abi.STAGE_CACHE)
        g.redecide(1.1, offered)
        g.ev = "config3 index"
        g.free(1.0)  # (the two decisions of the queue took every slot)
        head = 5000  # the first requests' leases, reported as running with their digests
        gr = g.solve(1.2, np.ascontiguousarray(q[:head]))
        _, dm = g.oracle.derive_task_keys(np.ascontiguousarray(q[:head]), TaskSources(
            src.args, src.args_offsets, src.args_index[:head], src.source_digests[:head]))
        index_from(g, dm, gr)
        g.ev = "config3 both stages"
        offered = g.filtered(2.0, q, cuts, srcs=srcs, stages=_abi.STAGE_CACHE | _abi.STAGE_DEDUPE)
        g.redecide(2.1, offered)
        g.free()
    except Mismatch:
        ok = False
    print(json.dumps({"case": "config3", "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    return ok


def main():
    a = ARGS
    ok = True
    if a.fuzz:
        ok = run_fuzz(a.world, a.fuzz, a.seed * 1000 + 1) and ok
    if a.config3:
        ok = run_config3(a.world, a.seed * 1000 + 2) and ok
    line = {"shard_filter": ok, "world": a.world, "nccl": "real" if FAKE is None else "fake_nccl",
            "torch_loaded": "torch" in sys.modules}
    print(json.dumps(line), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
