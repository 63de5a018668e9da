#!/usr/bin/env python
"""Parity of the range-sharded scheduler (include/ydshard.h) on ONE GPU: W rank handles in W threads of one process.

The ranks talk through tests/fake_nccl/libnccl.so.2, a test-only stand-in for the five NCCL calls the scheduler makes
(every collective is a host rendezvous that checks that all ranks made the same call).  It is loaded with RTLD_GLOBAL
before anything else, so the scheduler's dlopen("libnccl.so.2") resolves to it through the SONAME; this process must
not import torch, which loads the real library.  With --real-nccl the process imports torch first and runs ONE rank
over the real NCCL instead (the library's binding to it, which the stand-in cannot cover).

Every event of a stream goes to every rank handle and to one CPU checker handle (oracle/libydoracle.so) fed the
concatenated queue:
  wait / solve      the sharded solve; the queue is cut into W ranges at seeded cut points (even, uneven, empty
                    ranks, one-request ranks, local lengths around 1024), some ranks stage their range first
  free / free_frac  yd_shard_free_tasks; every id goes to a random rank, some to two ranks
  keepalive         every rank; the answer is the OR over ranks
  notify*           every rank; an id is unknown iff it is unknown on every rank
  running           every rank; the ranks' lists together (each keeps the reported tasks whose lease it holds)
  hb, tick          every rank
After every event each rank's grants must equal the checker's slice bit for bit, and every rank's servant state, the
next task id, the sum of the ranks' lease counts and the combined answers must equal the checker's.  running_tasks
(and capacity_available, which follows from it) is compared after events that made a collective call: a lease lives
on one rank only, so a zombie swept by a heartbeat lowers running_tasks on its holder at once and on the other ranks
at the next collective, which exchanges the ranks' local decrements before anything reads them.

Prints one JSON line per failure and a final {"shard_parity": ...} line; exit code 0 iff everything matched.
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE_NCCL = ROOT / "tests" / "fake_nccl" / "libnccl.so.2"
ORACLE = ROOT / "oracle" / "libydoracle.so"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--fuzz", default="", help="comma-separated fuzz_stream seeds")
    ap.add_argument("--unique-hosts", action="store_true")
    ap.add_argument("--config", default="", help="comma-separated config names (see CONFIGS)")
    ap.add_argument("--golden", action="store_true", help="cfg5-1m: check the reference's digest instead of the checker")
    ap.add_argument("--refusals", action="store_true")
    ap.add_argument("--real-nccl", action="store_true")
    ap.add_argument("--seed", type=int, default=0)
    return ap.parse_args()


ARGS = parse()
if ARGS.real_nccl:
    import torch  # noqa: F401  (its libnccl.so.2 is the one the scheduler's dlopen finds)
    FAKE = None
else:
    FAKE = C.CDLL(str(FAKE_NCCL), mode=C.RTLD_GLOBAL)
    FAKE.yd_fake_nccl_stats.argtypes = [C.c_int, C.POINTER(C.c_ulonglong)]
    FAKE.yd_fake_nccl_stats.restype = None

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT_DTYPE, REQ_DTYPE, STATUS_GRANTED, STATUS_TIMEOUT  # noqa: E402
from yadcc_b200.dispatcher import RunningTask, Servant, TaskDispatcher  # noqa: E402

if FAKE is not None:
    assert "torch" not in sys.modules, "torch loads the real libnccl.so.2"


def ns(now: float) -> int:
    return int(round(now * 1_000_000_000))


def par(fns):
    """Run fns in one thread each (ctypes releases the GIL); return their results in order."""
    out = [None] * len(fns)
    err = []

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


class Harness:
    def __init__(self, name: str, world: int, seed: int, oracle: bool = True):
        self.name, self.W = name, world
        self.rng = np.random.default_rng(seed)
        self.lib = _abi.load_library()
        self.ranks = [TaskDispatcher(self.lib) for _ in range(world)]
        self.oracle = TaskDispatcher(str(ORACLE)) if oracle else None
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        assert self.lib.yd_shard_unique_id(uid) == 0, "yd_shard_unique_id"
        rcs = par([lambda r=r: self.lib.yd_shard_init(self.ranks[r]._h, r, world, uid) for r in range(world)])
        assert rcs == [0] * world, f"yd_shard_init: {rcs}"
        self.pending = np.zeros(0, dtype=REQ_DTYPE)
        self.outstanding: dict[int, int] = {}
        self.counts = {"events": 0, "solves": 0, "frees": 0, "collectives": 0, "handbacks": 0, "retried": 0,
                       "max_merge_rounds": 0, "lazy_checks": 0}
        self.trace: list = []
        self.cuts: list = []
        self.ev = None

    def close(self):
        for d in self.ranks:
            self.lib.yd_shard_finalize(d._h)
            d.close()
        if self.oracle:
            self.oracle.close()

    # -- the stand-in's counters ---------------------------------------------------------------------------
    def fake_stats(self):
        if FAKE is None:
            return None
        out = []
        for r in range(self.W):
            a = (C.c_ulonglong * 4)()
            FAKE.yd_fake_nccl_stats(r, a)
            out.append(np.asarray(list(a), dtype=np.int64))
        return np.stack(out)

    def fail(self, what: str, **kw):
        line = {"case": self.name, "world": self.W, "event": self.counts["events"], "kind": self.ev[0] if self.ev else None,
                "error": what, "cuts": self.cuts}
        line.update(kw)
        print(json.dumps(line, default=int), flush=True)
        raise Mismatch(what)

    # -- cut points ------------------------------------------------------------------------------------------
    def cut_points(self, n: int):
        W, rng = self.W, self.rng
        kind = rng.choice(["even", "uneven", "empty-first", "empty-middle", "empty-last", "ones", "len1023", "len1024",
                           "len1025"])
        if kind == "even" or W == 1:
            c = [n * g // W for g in range(W + 1)]
        elif kind == "uneven":
            c = sorted(int(x) for x in rng.integers(0, n + 1, W - 1))
            c = [0] + c + [n]
        elif kind.startswith("empty"):
            e = {"empty-first": 0, "empty-middle": W // 2, "empty-last": W - 1}[kind]
            others = [g for g in range(W) if g != e]
            sizes = [0] * W
            for k, g in enumerate(others):
                sizes[g] = n * (k + 1) // len(others) - n * k // len(others)
            c = [0] + list(np.cumsum(sizes))
        elif kind == "ones":
            sizes = [min(1, n)] * W
            rest = n - sum(sizes)
            sizes[int(rng.integers(0, W))] += max(rest, 0)
            if rest < 0:
                sizes = [1 if g < n else 0 for g in range(W)]
            c = [0] + list(np.cumsum(sizes))
        else:
            m = int(kind[3:])
            g = int(rng.integers(0, W))
            sizes = [0] * W
            sizes[g] = min(m, n)
            left = n - sizes[g]
            others = [x for x in range(W) if x != g]
            for k, x in enumerate(others):
                sizes[x] = left * (k + 1) // len(others) - left * k // len(others)
            c = [0] + list(np.cumsum(sizes))
        c = [int(x) for x in c]
        assert c[0] == 0 and c[-1] == n and all(a <= b for a, b in zip(c, c[1:])), (kind, c, n)
        return c

    # -- events ---------------------------------------------------------------------------------------------------------
    def solve(self, now: float, full: np.ndarray) -> np.ndarray:
        W, n = self.W, len(full)
        cuts = self.cuts = self.cut_points(n)
        staged = self.rng.random(W) < 0.4
        parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(W)]
        for r in range(W):
            if staged[r]:  # the range, sometimes followed by unrelated requests
                q = parts[r]
                if self.rng.random() < 0.5 and n:
                    q = np.concatenate([q, full[: int(self.rng.integers(1, n + 1))]])
                self.ranks[r].stage_requests(np.ascontiguousarray(q))
        outs = [np.zeros(max(len(p), 1), dtype=GRANT_DTYPE) for p in parts]
        before = self.fake_stats()

        def call(r):
            p = parts[r]
            return self.lib.yd_shard_wait_for_starting_new_tasks(self.ranks[r]._h, ns(now), None if staged[r] else p.ctypes.data,
                                                                  len(p), outs[r].ctypes.data)
        rcs = par([lambda r=r: call(r) for r in range(W)])
        self.counts["solves"] += 1
        if any(rc != 0 for rc in rcs):
            self.fail("sharded solve did not decide the batch", rcs=rcs, staged=staged.tolist())
        g = np.concatenate([outs[r][: len(parts[r])] for r in range(W)]) if n else np.zeros(0, GRANT_DTYPE)
        if self.oracle is not None:
            g1 = self.oracle.wait_for_starting_new_tasks(np.ascontiguousarray(full), now).copy()
            bad = (g["status"] != g1["status"]) | (g["servant_index"] != g1["servant_index"]) | (g["task_id"] != g1["task_id"])
            if bad.any():
                i = int(np.nonzero(bad)[0][0])
                r = int(np.searchsorted(cuts, i, side="right") - 1)
                self.fail("grants differ", rank=r, index=i, local_index=i - cuts[r], mismatches=int(bad.sum()),
                          sharded=[int(x) for x in g[i]], single=[int(x) for x in g1[i]], staged=staged.tolist())
        self.check_solve_stats(before)
        ok = g["status"] == STATUS_GRANTED
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        return g

    def check_solve_stats(self, before):
        if before is None:
            return
        d = self.fake_stats() - before
        if not (d == d[0]).all():
            self.fail("ranks made different numbers of collectives", calls=d.tolist())
        calls, gathers, reduces, nbytes = (int(x) for x in d[0])
        self.counts["collectives"] += calls
        if calls == 0:
            return  # no servant or no digest: nothing to exchange
        st = _abi.yd_shard_stats()
        for r in range(self.W):
            if self.lib.yd_shard_last_stats(self.ranks[r]._h, C.byref(st)) != 1:
                continue  # (no batch decided by the sharded path yet)
            self.counts["max_merge_rounds"] = max(self.counts["max_merge_rounds"], int(st.merge_rounds))
            if gathers == 2 and reduces <= 2:  # one attempt, decided by the sharded path
                xb = [int(x) for x in st.exchange_bytes]
                if reduces != 1 + (xb[2] > 0) or int(d[r][3]) != sum(xb):
                    self.fail("exchange bytes differ from what the stand-in moved", rank=r, exchange_bytes=xb,
                              moved=int(d[r][3]), calls=d[r].tolist())
        if gathers % 2:
            self.counts["handbacks"] += 1  # the ranges' all-gather of a batch the sequential solver decided
        if gathers > 3:
            self.counts["retried"] += 1

    def free(self, ids: np.ndarray):
        W, rng = self.W, self.rng
        ids = np.asarray(ids, dtype=np.uint64)
        to = [[] for _ in range(W)]
        for x in ids.tolist():
            r = int(rng.integers(0, W))
            to[r].append(x)
            if W > 1 and rng.random() < 0.25:
                to[(r + 1 + int(rng.integers(0, W - 1))) % W].append(x)
        arrs = [np.ascontiguousarray(np.asarray(t, dtype=np.uint64)) for t in to]
        before = self.fake_stats()
        rcs = par([lambda r=r: self.lib.yd_shard_free_tasks(self.ranks[r]._h, arrs[r].ctypes.data if len(arrs[r]) else None,
                                                             len(arrs[r])) for r in range(W)])
        if any(rcs):
            self.fail("yd_shard_free_tasks failed", rcs=rcs)
        if self.oracle is not None:
            self.oracle.free_tasks(ids)
        self.counts["frees"] += 1
        if before is not None:
            d = self.fake_stats() - before
            S_ = self.ranks[0].num_servants()
            # the lengths, the ids (unless every list is empty), the running_tasks decrements
            gathers = 2 if len(ids) else 1
            if S_ and not ((d[:, 1] == gathers) & (d[:, 2] == 1)).all() or not S_ and d.any():
                self.fail("a collective free is two all-gathers and one all-reduce", calls=d.tolist())
            self.counts["collectives"] += int(d[0][0])
        for i in ids.tolist():
            self.outstanding.pop(i, None)

    def notify(self, loc: str, tasks):
        res = [d.notify_servant_running_tasks(loc, tasks) for d in self.ranks]
        common = set(res[0])
        for x in res[1:]:
            common &= set(x)
        mine = sorted(x for x in res[0] if x in common)
        if self.oracle is not None:
            want = sorted(self.oracle.notify_servant_running_tasks(loc, tasks))
            if mine != want:
                self.fail("unknown ids differ", sharded=mine[:20], single=want[:20], per_rank=[sorted(x)[:20] for x in res])

    def every(self, f):
        for d in self.ranks:
            f(d)
        if self.oracle is not None:
            f(self.oracle)

    def event(self, ev, build):
        """`build(kind_index, f)`: the value of a per-handle builder, checked equal on every handle."""
        self.ev = ev
        kind = ev[0]
        before = self.fake_stats()
        if kind == "hb":
            _, now, sv, exp = ev
            self.every(lambda d: d.keep_servant_alive(sv, exp, now=now))
        elif kind == "enqueue":
            self.pending = np.concatenate([self.pending, ev[1]])
        elif kind == "solve":
            g = self.solve(ev[1], self.pending)
            self.pending = self.pending[g["status"] == STATUS_TIMEOUT]
        elif kind == "wait":
            self.solve(ev[1], build(ev[2]) if callable(ev[2]) else ev[2])
        elif kind == "free":
            self.free(ev[1])
        elif kind == "free_frac":
            _, seed, frac, *spare = ev
            ids = np.fromiter(sorted(self.outstanding), dtype=np.uint64, count=len(self.outstanding))
            pick = ids[np.random.default_rng(seed).random(len(ids)) < frac]
            if spare:
                pick = pick[np.asarray([self.outstanding[i] not in spare[0] for i in pick.tolist()], dtype=bool)]
            self.free(pick)
        elif kind == "keepalive":
            _, now, ids, exp = ev
            ids = np.asarray(sorted(self.outstanding) if ids is None else ids, dtype=np.uint64)
            oks = [d.keep_tasks_alive(ids, exp, now=now) for d in self.ranks]
            ok = np.logical_or.reduce(oks) if oks else None
            if self.oracle is not None:
                want = self.oracle.keep_tasks_alive(ids, exp, now=now)
                if not (ok == want).all():
                    i = int(np.nonzero(ok != want)[0][0])
                    self.fail("keep-alive answers differ", index=i, id=int(ids[i]), sharded=bool(ok[i]), single=bool(want[i]))
                if sum(o.astype(int) for o in oks).max(initial=0) > 1:
                    self.fail("a lease is alive on two ranks")
        elif kind == "tick":
            self.every(lambda d: d.on_expiration_timer(now=ev[1]))
        elif kind == "notify":
            _, loc, tasks = ev
            self.notify(loc, [RunningTask(a, b, loc, c) for a, b, c in tasks])
        elif kind == "notify_own":
            _, sidx, drop_seed, extra = ev
            loc = (self.oracle or self.ranks[0]).servant_location(sidx)
            if loc is not None:
                own = sorted(t for t, s in self.outstanding.items() if s == sidx)
                rng = np.random.default_rng(drop_seed)
                own = [t for t in own if rng.random() < 0.8]
                ids = own + list(extra)
                self.notify(loc, [RunningTask(1000 + k, t, loc, f"{t:064x}") for k, t in enumerate(ids)])
        elif kind == "running":
            # a rank keeps the reported tasks whose lease it holds: the ranks' lists together are the single scheduler's
            key = lambda d: [(t.servant_task_id, t.task_grant_id, t.servant_location) for t in d.get_running_tasks()]  # noqa: E731
            mine = sorted(x for d in self.ranks for x in key(d))
            if self.oracle is not None and mine != sorted(key(self.oracle)):
                self.fail("running tasks differ", sharded=mine[:10], single=sorted(key(self.oracle))[:10])
        elif kind == "state":
            pass
        else:
            raise ValueError(kind)
        collective = before is None or bool((self.fake_stats() - before)[:, 0].any()) or self.W == 1
        self.compare(collective)
        self.counts["events"] += 1

    def compare(self, collective: bool):
        sts = [d.servant_state() for d in self.ranks]
        ref = self.oracle.servant_state() if self.oracle is not None else sts[0]
        fields = ["ever_assigned_tasks", "expires_at_ns"]
        if collective:
            fields += ["running_tasks", "capacity_available"]
        else:
            self.counts["lazy_checks"] += 1
        for r, st in enumerate(sts):
            if len(st) != len(ref):
                self.fail("servant counts differ", rank=r, sharded=len(st), single=len(ref))
            for f in fields:
                bad = np.nonzero(st[f] != ref[f])[0]
                if len(bad):
                    i = int(bad[0])
                    self.fail(f"{f} differs", rank=r, index=i, sharded=int(st[f][i]), single=int(ref[f][i]),
                              differing=int(len(bad)))
        ids = [d.next_task_id() for d in self.ranks]
        want = self.oracle.next_task_id() if self.oracle is not None else ids[0]
        if any(x != want for x in ids):
            self.fail("next_task_id differs", sharded=ids, single=want)
        if self.oracle is not None:
            alive = sum(d.num_tasks() for d in self.ranks)
            if alive != self.oracle.num_tasks():
                self.fail("sum of num_tasks differs", sharded=alive, single=self.oracle.num_tasks(),
                          per_rank=[d.num_tasks() for d in self.ranks])

    def run(self, streams_by_handle):
        """streams_by_handle[k]: the stream built on handle k (ranks, then the checker), so intern ids agree."""
        base = streams_by_handle[-1]
        handles = self.ranks + ([self.oracle] if self.oracle is not None else [])
        for k, ev in enumerate(base.events):
            for other in streams_by_handle[:-1]:
                e2 = other.events[k]
                if ev[0] in ("wait", "enqueue") and not callable(e2[-1]):
                    a, b = ev[-1], e2[-1]
                    assert a.shape == b.shape and (a == b).all(), "intern ids differ between handles"

            def build(f, k=k):
                vals = [streams_by_handle[h].events[k][2](handles[h]) for h in range(len(handles))]
                for v in vals[:-1]:
                    assert v.shape == vals[-1].shape and (v == vals[-1]).all(), "intern ids differ between handles"
                return vals[-1]
            self.event(ev, build)


# ---- cases ----------------------------------------------------------------------------------------------------------------
def workload_stream(w: S.Workload, d: TaskDispatcher, rounds: int = 2) -> S.Stream:
    """Register, then `rounds` x (the whole queue, a collective free of a seeded half of the grants, a tick)."""
    ev: list = [("hb", 0.0, sv, 3600.0) for sv in w.servants]
    full = w.build_requests(d)
    for rnd in range(rounds):
        now = 0.001 + rnd
        ev += [("wait", now, full), ("free_frac", 100 + rnd, 0.5), ("tick", now + 0.5), ("state",)]
    return S.Stream(w.name, ev)


def class_bound_workload() -> S.Workload:
    """cfg2-mod's servants (8 independent components), min_version 0..5: 48 classes overflow the first class bound."""
    w = S.config2(4000, 160, 8, variant="mod")
    inner = w.build_requests

    def build(d):
        r = inner(d)
        r["min_version"] = np.random.default_rng(5).integers(0, 6, len(r)).astype(np.uint32)
        return r
    return S.Workload("class-bound", w.servants, w.digests, build)


CONFIGS = {
    "cfg2-mod-small": lambda: S.config2(5000, 200, 8, variant="mod"),
    "cfg2-random-small": lambda: S.config2(5000, 200, 8, variant="random"),
    "cfg-self-small": lambda: S.config_self(6000, 150),
    "cfg3-20k": lambda: S.config3(20000, 300, 8),
    "cfg2-mod": lambda: S.config2(variant="mod"),
    "cfg2-random": lambda: S.config2(variant="random"),
    "cfg-self": lambda: S.config_self(),
    "class-bound": class_bound_workload,
}


def make_handles_streams(h: Harness, make):
    handles = h.ranks + ([h.oracle] if h.oracle is not None else [])
    return [make(d) for d in handles]


def run_case(name, world, make, seed, oracle=True):
    h = Harness(name, world, seed, oracle)
    try:
        h.run(make_handles_streams(h, make))
        ok = True
    except Mismatch:
        ok = False
    line = {"case": name, "world": world, "ok": ok}
    line.update(h.counts)
    print(json.dumps(line), flush=True)
    return h, ok


def golden_case(world):
    """cfg5-1m's first solve over `world` ranks against the digest the reference's own scheduler produced."""
    golden = json.loads((ROOT / "tests" / "golden" / "digests.json").read_text())["streams"]["cfg5-1m"]
    w = S.config5(1_000_000, 8000)
    h = Harness("cfg5-1m", world, 7, oracle=False)
    ok = True
    try:
        fulls = [w.build_requests(d) for d in h.ranks]
        for f in fulls[1:]:
            assert (f == fulls[0]).all()
        h.every(lambda d: [d.keep_servant_alive(sv, 10.0, now=0.0) for sv in w.servants])
        g = h.solve(0.001, fulls[0])
        h.ev = ("state",)
        h.compare(True)
        st = h.ranks[0].servant_state()
        for r, d in enumerate(h.ranks[1:], 1):
            if not (d.servant_state()["running_tasks"] == st["running_tasks"]).all():
                h.fail("running_tasks differ between ranks", rank=r)
        trace = [g, np.stack([st["running_tasks"], st["ever_assigned_tasks"], st["capacity_available"]], axis=1),
                 np.asarray([h.ranks[0].next_task_id(), sum(d.num_tasks() for d in h.ranks), h.ranks[0].num_servants()],
                            dtype=np.uint64)]
        if S.trace_digest(trace) != golden["sha256"]:
            h.fail("cfg5-1m digest differs from the reference's")
    except Mismatch:
        ok = False
    print(json.dumps({"case": "cfg5-1m", "world": world, "ok": ok, "reference_digest_equal": ok, **h.counts}), flush=True)
    h.close()
    return ok


def refusal_case(world):
    """A cluster with capacities above the narrow key limit returns 1 on every rank and changes nothing; so does a staged
    solve that asks for more requests than were staged."""
    h = Harness("refusals", world, 3, oracle=False)
    ok = True
    try:
        dg = "ab" * 32
        sv = Servant("10.9.0.1:8000", None, [dg], 8, 40000, 0, 64 << 30, 40 << 30, 70000, _abi.PRIORITY_USER)
        small = Servant("10.9.0.2:8000", None, [dg], 8, 8, 0, 64 << 30, 40 << 30, 4, _abi.PRIORITY_USER)
        h.every(lambda d: d.keep_servant_alive(small, 100.0, now=0.0))
        env = [d.intern_env(dg) for d in h.ranks]
        ip = [d.intern_ip("172.16.0.1") for d in h.ranks]
        reqs = [S._requests(d, np.full(3, env[r], np.uint32), np.full(3, ip[r], np.uint32), 8) for r, d in enumerate(h.ranks)]
        # staged queue shorter than asked for
        for r, d in enumerate(h.ranks):
            d.stage_requests(np.ascontiguousarray(reqs[r][:1]))
        before = (h.fake_stats(), [d.next_task_id() for d in h.ranks], [d.servant_state().copy() for d in h.ranks])
        out = np.zeros(4, dtype=GRANT_DTYPE)
        rcs = par([lambda r=r: h.lib.yd_shard_wait_for_starting_new_tasks(h.ranks[r]._h, ns(0.1), None, 3, out.ctypes.data)
                   for r in range(world)])
        if rcs != [1] * world:
            h.fail("a staged solve longer than the staged queue was not refused", rcs=rcs)
        h.every(lambda d: d.keep_servant_alive(sv, 100.0, now=0.2))
        outs = [np.zeros(3, dtype=GRANT_DTYPE) for _ in range(world)]
        rcs = par([lambda r=r: h.lib.yd_shard_wait_for_starting_new_tasks(h.ranks[r]._h, ns(0.3), reqs[r].ctypes.data, 3,
                                                                        outs[r].ctypes.data) for r in range(world)])
        if rcs != [1] * world:
            h.fail("a wide cluster was not refused", rcs=rcs)
        after = h.fake_stats()
        if before[0] is not None and (after - before[0]).any():
            h.fail("a refused solve made a collective call")
        for r, d in enumerate(h.ranks):
            st = d.servant_state()
            if d.next_task_id() != before[1][r] or d.num_tasks() != 0 or st["running_tasks"].any() \
                    or st["ever_assigned_tasks"].any():
                h.fail("a refused solve changed the state", rank=r)
    except Mismatch:
        ok = False
    print(json.dumps({"case": "refusals", "world": world, "ok": ok}), flush=True)
    h.close()
    return ok


def main():
    a = ARGS
    ok = True
    cases = []
    for s in [int(x) for x in a.fuzz.split(",") if x]:
        cases.append((f"fuzz-{s}" + ("-unique" if a.unique_hosts else ""),
                      lambda d, s=s: S.fuzz_stream(d, s, n_servants=8 + s % 30, unique_hosts=a.unique_hosts)))
    for c in [x for x in a.config.split(",") if x]:
        cases.append((c, lambda d, c=c: workload_stream(CONFIGS[c](), d)))
    for k, (name, make) in enumerate(cases):
        h, good = run_case(name, a.world, make, a.seed * 1000 + k)
        h.close()
        ok = ok and good
    if a.golden:
        ok = golden_case(a.world) and ok
    if a.refusals:
        ok = refusal_case(a.world) and ok
    line = {"shard_parity": ok, "world": a.world, "nccl": "real" if FAKE is None else "fake_nccl"}
    if FAKE is not None:
        a4 = (C.c_ulonglong * 4)()
        FAKE.yd_fake_nccl_stats(0, a4)
        line["fake_nccl_collectives"] = int(a4[0])
        line["torch_loaded"] = "torch" in sys.modules
    print(json.dumps(line), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
