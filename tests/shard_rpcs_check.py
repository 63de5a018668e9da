#!/usr/bin/env python
"""The replicated calls of the range-sharded scheduler (include/ydshard.h) on ONE GPU: W rank handles in W threads of
one process, over the test-only NCCL stand-in (tests/fake_nccl/libnccl.so.2, loaded with RTLD_GLOBAL before anything
else; this process must not import torch).  With --real-nccl the process imports torch first and runs one rank over
the real NCCL.

Each replicated call is made by every rank with the same arguments, and EVERY rank's answer must equal, exactly, the
answer of one CPU checker handle (oracle/libydoracle.so) fed the concatenated queue:
  --fuzz      streams.fuzz_stream: keep-alive flags, unknown ids in request order with per-item counts, running tasks in
              order with all four fields, the in-flight index after a group refresh; running_tasks after every call
  --rpcs      seeded windows of WaitForStartingTask RPCs: results and grants
  --service   W group services (yd_shard_service_create) fed the frames of tests/wire_cases.py's scenario and a random
              request stream: every rank's bytes equal one yd_service_create service's over the checker; with
              token_seed 0 every rank hands out the same tokens

Prints one JSON line per case and a final {"shard_rpcs": ...} line; exit code 0 iff everything matched.
"""
import argparse
import ctypes as C
import json
import sys
import threading
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE_NCCL = ROOT / "tests" / "fake_nccl" / "libnccl.so.2"
ORACLE = ROOT / "oracle" / "libydoracle.so"

ap = argparse.ArgumentParser()
ap.add_argument("--world", type=int, default=2)
ap.add_argument("--fuzz", default="", help="comma-separated fuzz_stream seeds")
ap.add_argument("--unique-hosts", action="store_true")
ap.add_argument("--rpcs", type=int, default=0, help="number of seeded RPC windows")
ap.add_argument("--service", action="store_true")
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
sys.path.insert(0, str(ROOT / "tests"))
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT_DTYPE, RPC_WAIT_DTYPE, STATUS_GRANTED, STATUS_TIMEOUT  # noqa: E402
from yadcc_b200.dispatcher import RunningTask, Servant, TaskDispatcher  # noqa: E402

if FAKE is not None:
    assert "torch" not in sys.modules, "torch loads the real libnccl.so.2"


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


class Group:
    """W rank handles joined to one group, and the checker."""

    def __init__(self, name: str, world: int, seed: int):
        self.name, self.W = name, world
        self.rng = np.random.default_rng(seed)
        self.lib = _abi.load_library()
        self.ranks = [TaskDispatcher(self.lib) for _ in range(world)]
        self.oracle = TaskDispatcher(str(ORACLE))
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        assert self.lib.yd_shard_unique_id(uid) == 0, "yd_shard_unique_id"
        rcs = par([lambda r=r: self.lib.yd_shard_init(self.ranks[r]._h, r, world, uid) for r in range(world)])
        assert rcs == [0] * world, f"yd_shard_init: {rcs}"
        self.counts = {"events": 0, "keepalive": 0, "notify": 0, "running": 0, "index": 0, "rpc_windows": 0,
                       "refusals": 0}
        self.outstanding: dict[int, int] = {}
        self.ev = None

    def close(self):
        for d in self.ranks:
            self.lib.yd_shard_finalize(d._h)
            d.close()
        self.oracle.close()

    def fail(self, what: str, **kw):
        line = {"case": self.name, "world": self.W, "event": self.counts["events"], "kind": self.ev, "error": what}
        line.update(kw)
        print(json.dumps(line, default=str), flush=True)
        raise Mismatch(what)

    def every(self, f):
        for d in self.ranks + [self.oracle]:
            f(d)

    def same(self, what, got, want, **kw):
        for r, g in enumerate(got):
            if g != want:
                self.fail(f"{what} differ", rank=r, group=str(g)[:400], single=str(want)[:400], **kw)

    # -- the calls -----------------------------------------------------------------------------------------------------
    def solve(self, now, full):
        n, W = len(full), self.W
        cuts = [n * g // W for g in range(W + 1)]
        parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(W)]
        outs = [np.zeros(max(len(p), 1), dtype=GRANT_DTYPE) for p in parts]
        rcs = par([lambda r=r: self.lib.yd_shard_wait_for_starting_new_tasks(
            self.ranks[r]._h, ns(now), parts[r].ctypes.data, len(parts[r]), outs[r].ctypes.data) for r in range(W)])
        if any(rcs):
            self.fail("sharded solve refused", rcs=rcs)
        g = np.concatenate([outs[r][:len(parts[r])] for r in range(W)]) if n else np.zeros(0, GRANT_DTYPE)
        g1 = self.oracle.wait_for_starting_new_tasks(np.ascontiguousarray(full), now).copy()
        for k in ("status", "servant_index", "task_id"):
            if not (g[k] == g1[k]).all():
                self.fail("grants differ", field=k)
        ok = g["status"] == STATUS_GRANTED
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        return g

    def free(self, ids):
        ids = np.ascontiguousarray(np.asarray(ids, dtype=np.uint64))
        empty = np.zeros(0, dtype=np.uint64)
        args = [ids if r == 0 else empty for r in range(self.W)]
        rcs = par([lambda r=r: self.lib.yd_shard_free_tasks(self.ranks[r]._h, args[r].ctypes.data if len(args[r]) else None,
                                                             len(args[r])) for r in range(self.W)])
        if any(rcs):
            self.fail("yd_shard_free_tasks failed", rcs=rcs)
        self.oracle.free_tasks(ids)
        for i in ids.tolist():
            self.outstanding.pop(i, None)

    def keepalive(self, now, ids, exp):
        ids = np.ascontiguousarray(np.asarray(ids, dtype=np.uint64))
        got = par([lambda d=d: d._keep_alive_with(self.lib.yd_shard_keep_task_alive, ids, exp, now).tolist()
                   for d in self.ranks])
        self.same("keep-alive flags", got, self.oracle.keep_tasks_alive(ids, exp, now=now).tolist())
        self.counts["keepalive"] += 1

    def notify(self, batch):
        got = par([lambda d=d: d._notify_with(self.lib.yd_shard_notify_servants_running_tasks, batch) for d in self.ranks])
        self.same("unknown ids", got, self.oracle.notify_servants_running_tasks(batch), items=len(batch))
        self.counts["notify"] += 1

    def running(self):
        got = par([lambda d=d: d._running_with(self.lib.yd_shard_get_running_tasks) for d in self.ranks])
        want = self.oracle.get_running_tasks()
        self.same("running tasks", got, want)
        self.counts["running"] += 1
        # the in-flight index over the group's list, probed on every rank
        n = par([lambda d=d: int(self.lib.yd_shard_running_index_refresh(d._h)) for d in self.ranks])
        self.same("index sizes", n, self.oracle.running_index_refresh())
        keys = sorted({t.task_digest for t in want if len(t.task_digest) == 64} | {f"{k:064x}" for k in range(4)})
        hits = [d.find_running_tasks(keys) for d in self.ranks]
        ref = self.oracle.find_running_tasks(keys)
        self.same("index hits", [h.tolist() for h in hits], ref.tolist())
        self.counts["index"] += 1

    def compare(self):
        ref = self.oracle.servant_state()
        for r, d in enumerate(self.ranks):
            st = d.servant_state()
            if len(st) != len(ref):
                self.fail("servant counts differ", rank=r)
            for f in ("running_tasks", "ever_assigned_tasks", "capacity_available", "expires_at_ns"):
                bad = np.nonzero(st[f] != ref[f])[0]
                if len(bad):
                    self.fail(f"{f} differs", rank=r, index=int(bad[0]), group=int(st[f][bad[0]]), single=int(ref[f][bad[0]]))
            if d.next_task_id() != self.oracle.next_task_id():
                self.fail("next_task_id differs", rank=r)
        if sum(d.num_tasks() for d in self.ranks) != self.oracle.num_tasks():
            self.fail("sum of num_tasks differs")


# ---- fuzz streams ---------------------------------------------------------------------------------------------------------
def run_fuzz(seed: int, world: int, unique: bool, case_seed: int) -> bool:
    name = f"fuzz-{seed}" + ("-unique" if unique else "")
    g = Group(name, world, case_seed)
    handles = g.ranks + [g.oracle]
    streams = [S.fuzz_stream(d, seed, n_servants=8 + seed % 30, unique_hosts=unique) for d in handles]
    pending = np.zeros(0, dtype=_abi.REQ_DTYPE)
    ok = True
    try:
        for k, ev in enumerate(streams[-1].events):
            g.ev = ev[0]
            kind = ev[0]
            if kind == "hb":
                g.every(lambda d: d.keep_servant_alive(ev[2], ev[3], now=ev[1]))
            elif kind == "tick":
                g.every(lambda d: d.on_expiration_timer(now=ev[1]))
            elif kind == "enqueue":
                pending = np.concatenate([pending, ev[1]])
            elif kind == "solve":
                gr = g.solve(ev[1], pending)
                pending = pending[gr["status"] == STATUS_TIMEOUT]
            elif kind == "wait":
                # a builder interns on each handle, as the stream was built on each
                q = [st.events[k][2](h) for st, h in zip(streams, handles)][-1] if callable(ev[2]) else ev[2]
                g.solve(ev[1], q)
            elif kind == "free":
                g.free(ev[1])
            elif kind == "free_frac":
                _, fs, frac, *spare = ev
                ids = np.fromiter(sorted(g.outstanding), dtype=np.uint64, count=len(g.outstanding))
                pick = ids[np.random.default_rng(fs).random(len(ids)) < frac]
                if spare:
                    pick = pick[np.asarray([g.outstanding[i] not in spare[0] for i in pick.tolist()], dtype=bool)]
                g.free(pick)
            elif kind == "keepalive":
                _, now, ids, exp = ev
                ids = sorted(g.outstanding) + [10**12] if ids is None else ids
                g.keepalive(now, ids, exp)
            elif kind in ("notify", "notify_own"):
                if kind == "notify":
                    loc, tasks = ev[1], [RunningTask(a, b, ev[1], c) for a, b, c in ev[2]]
                else:
                    _, sidx, drop_seed, extra = ev
                    loc = g.oracle.servant_location(sidx)
                    if loc is None:
                        loc = "10.255.0.1:1"
                    own = sorted(t for t, s in g.outstanding.items() if s == sidx)
                    r2 = np.random.default_rng(drop_seed)
                    own = [t for t in own if r2.random() < 0.8]
                    tasks = [RunningTask(1000 + j, t, loc, f"{t:064x}") for j, t in enumerate(own + list(extra))]
                batch = [(loc, tasks)]
                x = g.rng.random()
                if x < 0.2:
                    batch = [(loc, tasks), (loc, tasks[::2])]  # the same servant twice: the batch is cut there
                elif x < 0.4 and g.oracle.num_servants():
                    other = g.oracle.servant_location(int(g.rng.integers(0, g.oracle.num_servants())))
                    batch = [(loc, tasks), (other, [])]
                g.notify(batch)
            elif kind == "running":
                g.running()
            elif kind == "state":
                pass
            else:
                raise ValueError(kind)
            g.compare()
            g.counts["events"] += 1
        g.running()
    except Mismatch:
        ok = False
    print(json.dumps({"case": name, "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    return ok


# ---- RPC windows ------------------------------------------------------------------------------------------------------------
def run_rpcs(n_windows: int, world: int, case_seed: int) -> bool:
    g = Group("rpc-windows", world, case_seed)
    rng = g.rng
    digests = [f"{i:02x}" * 32 for i in range(5)]
    servants = []
    for i in range(24):
        host = f"10.3.0.{i % 16}"  # 8 hosts with two servants: a requestor there needs the sequential solver
        envs = [digests[i % 4]] + ([digests[4]] if i % 5 == 0 else [])
        servants.append(Servant(f"{host}:{8000 + i}", None, envs, 8, 8, int(rng.integers(0, 3)), 64 << 30, 48 << 30,
                                int(rng.choice([2, 4, 8])), _abi.PRIORITY_USER if i % 3 else _abi.PRIORITY_DEDICATED))
    ok = True
    try:
        g.every(lambda d: [d.keep_servant_alive(sv, 3600.0, now=0.0) for sv in servants])
        unknown = "ee" * 32
        bound = int(g.lib.yd_grant_capacity_bound(g.ranks[0]._h))
        for w in range(n_windows):
            g.ev = f"window {w}"
            now = 1.0 + w
            n = int(rng.choice([1, 2, 3, 7, 20, 60]))
            rows = []
            for _ in range(n):
                dg = digests[int(rng.integers(0, 5))] if rng.random() < 0.85 else unknown
                ip = f"10.3.0.{int(rng.integers(0, 16))}" if rng.random() < 0.3 else f"172.20.0.{int(rng.integers(0, 9))}"
                imm = int(rng.choice([0, 1, 1, 2, 4, bound + 5, 0xFFFFFFFF]))
                pre = int(rng.choice([0, 0, 1, 3, bound * 2]))
                ms = int(rng.choice([0, 100, 10000, 10001]))
                ka = int(rng.choice([1, 10, 30, 31])) * 1_000_000_000
                rows.append((dg, int(rng.integers(0, 10)), ip, imm, pre, ms, ka))
            if w % 7 == 3:  # fewer decisions than ranks
                rows = rows[:1]
                rows[0] = (digests[0], 0, "172.20.0.1", 1, 0, 0, 10_000_000_000)

            def arr(d):
                r = np.zeros(len(rows), dtype=RPC_WAIT_DTYPE)
                for i, (dg, mv, ip, imm, pre, ms, ka) in enumerate(rows):
                    r[i] = (d.intern_env(dg), mv, d.intern_ip(ip), imm, pre, ms, ka)
                return r
            per = [arr(d) for d in g.ranks]
            want_res, want_gr = g.oracle.wait_for_starting_task_rpcs(arr(g.oracle), now)
            got = par([lambda r=r: g.ranks[r]._rpcs_with(g.lib.yd_shard_wait_for_starting_task_rpcs, per[r], now)
                       for r in range(world)])
            key = lambda res, gr: (res.tolist(), gr.tolist())  # noqa: E731
            g.same("RPC results and grants", [key(*x) for x in got], key(want_res, want_gr))
            for gr in want_gr.tolist():
                g.outstanding[int(gr[0])] = int(gr[1])
            g.counts["rpc_windows"] += 1
            g.compare()
            if w % 5 == 4:  # a cap one short of the window's decisions: every rank refuses, nothing is decided
                total = int(g.lib.yd_rpc_expanded_requests(g.ranks[0]._h, per[0].ctypes.data, len(rows)))
                if total:
                    res = [np.zeros(len(rows), dtype=_abi.RPC_RESULT_DTYPE) for _ in range(world)]
                    grs = [np.zeros(total, dtype=GRANT_DTYPE) for _ in range(world)]
                    before = g.oracle.next_task_id()
                    rcs = par([lambda r=r: g.lib.yd_shard_wait_for_starting_task_rpcs(
                        g.ranks[r]._h, ns(now), per[r].ctypes.data, len(rows), res[r].ctypes.data, grs[r].ctypes.data,
                        total - 1) for r in range(world)])
                    if rcs != [(1 << 64) - 1] * world:
                        g.fail("a window larger than cap was not refused", rcs=rcs)
                    if any(d.next_task_id() != before for d in g.ranks):
                        g.fail("a refused window decided something")
                    g.counts["refusals"] += 1
            if g.outstanding and rng.random() < 0.5:
                ids = sorted(g.outstanding)
                g.free([ids[i] for i in rng.choice(len(ids), size=len(ids) // 2, replace=False)])
                g.compare()
            if w % 4 == 1:
                g.keepalive(now + 0.5, sorted(g.outstanding)[:50] + [10**9], 5.0)
                g.compare()
            if w % 6 == 5:
                g.every(lambda d: d.on_expiration_timer(now=now + 0.6))
                g.compare()
    except Mismatch:
        ok = False
    print(json.dumps({"case": "rpc-windows", "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    return ok


# ---- services and the wire layer -----------------------------------------------------------------------------------------------
def run_service(world: int, case_seed: int) -> bool:
    from yadcc_b200.service import HeartbeatRequest, SchedulerService

    import wire_cases

    ok = True
    # 1. the wire scenario, recorded on a service over the checker, replayed on W group services
    calls = []

    class Recorder(SchedulerService):
        def handle_frames(self, frames, *, now=0.0, out_cap=None):
            out = super().handle_frames(frames, now=now, out_cap=out_cap)
            calls.append(("frames", list(frames), now, out))
            return out

        def call(self, method, body, remote_ip, *, now=0.0, remote_is_ipv6=False):
            out = super().call(method, body, remote_ip, now=now, remote_is_ipv6=remote_is_ipv6)
            calls.append(("call", (method, body, remote_ip), now, out))
            return out

    def services(make_dispatcher, kind):
        mk = lambda cls: cls(make_dispatcher(kind), acceptable_user_tokens="usr", acceptable_servant_tokens="srv",  # noqa: E731
                             token_seed=9, now=0.0)
        return mk(Recorder), mk(SchedulerService)

    keep = []

    def make_dispatcher(kind):
        d = TaskDispatcher(str(ORACLE))
        keep.append(d)
        return d
    wire_cases._services = services
    wire_cases.run_wire_scenario(make_dispatcher, "port")

    g = Group("service-wire", world, case_seed)
    try:
        svcs = par([lambda d=d: SchedulerService(_GroupView(d), acceptable_user_tokens="usr", acceptable_servant_tokens="srv",
                                                 token_seed=9, now=0.0) for d in g.ranks])
        for k, (kind, args, now, want) in enumerate(calls):
            g.ev = f"wire {kind} {k}"
            if kind == "frames":
                got = par([lambda s=s: s.handle_frames(args, now=now) for s in svcs])
            else:
                got = par([lambda s=s: s.call(*args, now=now) for s in svcs])
            g.same("wire responses", got, want)
        n_wire = len(calls)
        for s in svcs:
            s.close()
        g.close()

        # 2. a random request stream: every rank's answers equal one service's over the checker (a fresh group)
        g = Group("service-wire", world, case_seed + 1)
        one = SchedulerService(g.oracle, acceptable_user_tokens="u1,u2", acceptable_servant_tokens="s1,u2",
                               serving_daemon_token_rollout_interval=3, token_seed=case_seed + 1)
        svcs = par([lambda d=d: SchedulerService(_GroupView(d), acceptable_user_tokens="u1,u2", acceptable_servant_tokens="s1,u2",
                                                 serving_daemon_token_rollout_interval=3, token_seed=case_seed + 1)
                    for d in g.ranks])
        n_ops = _service_stream(g, svcs, one, HeartbeatRequest)
        one.close()
        for s in svcs:
            s.close()

        # 3. token_seed 0: the kernel's random tokens, the same on every rank, at creation and after a roll-out
        g.ev = "tokens"
        svcs = par([lambda d=d: SchedulerService(_GroupView(d), acceptable_user_tokens="u", acceptable_servant_tokens="s",
                                                 serving_daemon_token_rollout_interval=2) for d in g.ranks])
        seen = set()
        for now in (0.0, 2.5, 2.6, 5.5):
            got = par([lambda s=s: s.get_config("u", now=now) for s in svcs])
            g.same("random serving-daemon tokens", got, got[0])
            seen.add(got[0][1])
        if len(seen) != 3:
            g.fail("token roll-outs", seen=sorted(seen))
        for s in svcs:
            s.close()
    except Mismatch:
        ok = False
        n_wire = n_ops = 0
    print(json.dumps({"case": "service-wire", "world": world, "ok": ok, "wire_calls": n_wire, "service_ops": n_ops}),
          flush=True)
    g.close()
    for d in keep:
        d.close()
    return ok


class _GroupView:
    """What SchedulerService needs of a RangeShardedDispatcher, without torch: the rank handle, joined to the group."""

    native = True

    def __init__(self, local):
        self.local = local


def _service_stream(g: Group, svcs, one, HeartbeatRequest, n_ops: int = 300) -> int:
    rng = g.rng
    digests = [f"{i:02x}" * 32 for i in range(4)]
    granted: list[int] = []
    now = 0.0

    def all_same(what, f):
        got = par([lambda s=s: f(s) for s in svcs])
        want = f(one)
        g.same(what, got, want)
        return want

    for step in range(n_ops):
        now += float(rng.choice([0.0, 0.05, 0.4, 1.1, 2.6]))
        op = str(rng.choice(["hb", "hb", "hb", "wait", "wait", "batch", "keep", "free", "config", "running", "tick"]))
        g.ev = f"service {op} {step}"
        if op == "hb":
            k = int(rng.integers(0, 12))
            ip = f"10.7.0.{k}"
            loc = str(rng.choice([f"{ip}:8335", f"{ip}:8335", f"{ip}:8336", "nonsense"]))
            running = []
            if granted and rng.random() < 0.6:
                for t in rng.choice(granted, size=min(len(granted), 4), replace=False):
                    running.append(RunningTask(int(rng.integers(1, 99)), int(t), loc, f"{int(t):064x}"))
            if rng.random() < 0.3:
                running.append(RunningTask(7, int(rng.integers(10**6, 10**7)), loc, "ee" * 32))
            req = HeartbeatRequest(
                token=str(rng.choice(["u1", "s1", "s1", "bad"])), location=loc, remote_ip=ip,
                next_heartbeat_in_ms=int(rng.choice([0, 1000, 5000, 30000])), version=3, num_processors=16,
                current_load=int(rng.integers(0, 6)), servant_priority=int(rng.choice([1, 2])), capacity=int(rng.choice([2, 8])),
                total_memory_in_bytes=64 << 30, memory_available_in_bytes=32 << 30,
                env_digests=[digests[j] for j in rng.choice(4, size=int(rng.integers(1, 4)), replace=False)],
                running_tasks=running)
            all_same("heartbeat responses", lambda s: s.heartbeat(req, now=now))
        elif op in ("wait", "batch"):
            n_rpc = 1 if op == "wait" else int(rng.integers(2, 6))
            toks, rows = [], []
            for _ in range(n_rpc):
                toks.append(str(rng.choice(["u1", "u1", "u2", "s1", "bad"])))
                dg = digests[int(rng.integers(0, 4))] if rng.random() < 0.9 else "77" * 32
                ip = f"10.7.0.{int(rng.integers(0, 12))}" if rng.random() < 0.4 else "172.16.3.3"
                rows.append((dg, int(rng.integers(0, 4)), ip, int(rng.choice([0, 1, 1, 2, 5])), int(rng.choice([0, 0, 1, 3])),
                             int(rng.choice([0, 100, 10000, 10001])), int(rng.choice([1, 15, 30, 31])) * 1_000_000_000))

            def wait(s):
                d = s.dispatcher
                r = np.zeros(n_rpc, dtype=RPC_WAIT_DTYPE)
                for i, (dg, mv, ip, imm, pre, wait_ms, ka) in enumerate(rows):
                    r[i] = (d.intern_env(dg), mv, d.intern_ip(ip), imm, pre, wait_ms, ka)
                res, gr = s.wait_for_starting_tasks(toks, r, now=now)
                return res.tolist(), gr.tolist()
            _, gr = all_same("WaitForStartingTask answers", wait)
            granted.extend(int(x[0]) for x in gr)
        elif op == "keep" and granted:
            ids = [int(x) for x in rng.choice(granted, size=min(len(granted), 4), replace=False)] + [10**9]
            tok, ms = str(rng.choice(["u1", "s1"])), int(rng.choice([1000, 30000, 30001]))
            all_same("KeepTaskAlive answers", lambda s: [x.tolist() if hasattr(x, "tolist") else x
                                                         for x in s.keep_task_alive(tok, ids, ms, now=now)])
        elif op == "free" and granted:
            ids = [int(x) for x in rng.choice(granted, size=min(len(granted), 5), replace=False)]
            tok = str(rng.choice(["u1", "u1", "bad"]))
            all_same("FreeTask answers", lambda s: s.free_task(tok, ids))
        elif op == "config":
            tok = str(rng.choice(["u1", "u2", "s1"]))
            all_same("GetConfig answers", lambda s: s.get_config(tok, now=now))
        elif op == "running":
            all_same("GetRunningTasks answers", lambda s: s.get_running_tasks())
        elif op == "tick":
            g.every(lambda d: d.on_expiration_timer(now=now))
        g.compare()
    return n_ops


def main():
    a = ARGS
    ok = True
    k = 0
    for s in [int(x) for x in a.fuzz.split(",") if x]:
        ok = run_fuzz(s, a.world, a.unique_hosts, a.seed * 1000 + k) and ok
        k += 1
    if a.rpcs:
        ok = run_rpcs(a.rpcs, a.world, a.seed * 1000 + 500) and ok
    if a.service:
        ok = run_service(a.world, a.seed * 1000 + 700) and ok
    line = {"shard_rpcs": ok, "world": a.world, "nccl": "real" if FAKE is None else "fake_nccl",
            "torch_loaded": "torch" in sys.modules}
    print(json.dumps(line), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
