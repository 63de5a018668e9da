"""Seeded synthetic event streams for the scheduler hot path (SURVEY.md 8(d)).

A *stream* is a list of events; `Replayer.run` feeds them to any backend that
speaks the ydsched C ABI and returns a *trace* (one numpy array per event that
produces output).  Two backends are at parity iff their traces are equal
element-wise; `trace_digest` folds a trace into one SHA-256 for large runs.

Event kinds (tuples, first element is the kind):

  ("hb", now, Servant, expires_in)            one KeepServantAlive
  ("enqueue", REQ array)                      append to the FIFO pending queue
  ("solve", now)                              offer the whole pending queue in order
                                              (zero-wait); Timeout requests stay
                                              pending, everything else leaves
  ("wait", now, REQ array | f(dispatcher))    one-shot batch, no pending queue (f builds it when the event runs:
                                              requestor IPs interned between solves)
  ("free", ids)                               FreeTask per id
  ("free_frac", seed, frac[, spare])          free a seeded subset of outstanding grants (except those on the
                                              servant indices in `spare`)
  ("keepalive", now, ids | None, expires_in)  KeepTaskAlive (None = all outstanding)
  ("tick", now)                               OnExpirationTimer
  ("notify", location, [(servant_task_id, grant_id, digest)])
  ("notify_own", servant_index, drop_seed, extra_ids)
                                              heartbeat reporting the grants this
                                              servant holds (minus a seeded few, plus
                                              some bogus ids)
  ("running",)                                GetRunningTasks
  ("state",)                                  per-servant bookkeeping snapshot
  ("filter", now, REQ array, cache_keys, task_digests)
                                              one yd_filter_and_wait_for_starting_new_tasks call (keys: strings or
                                              uint8 matrices, or None to skip that stage); traces the verdicts, the
                                              in-flight hits and the grants of the offered requests

Task ids are the ordinal of the grant (the reference starts at 0 and increments
per grant, task_dispatcher.h:218, .cc:127), so "free"/"keepalive" events can
name ids before the stream is run.

The request distributions for the five BASELINE.json configs are built by
`config1` .. `config5`; `fuzz_stream` mixes every quirk at small scale.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field, replace
from typing import Any, Callable, Sequence

import numpy as np

from . import _abi
from ._abi import GRANT_DTYPE, REQ_DTYPE, STATUS_GRANTED, STATUS_TIMEOUT
from .dispatcher import RunningTask, Servant, TaskDispatcher

GiB = 1 << 30


def hex_digest(rng: np.random.Generator) -> str:
    """A BLAKE3-looking compiler digest: 64 lowercase hex chars (env_desc.proto:27-28)."""
    return rng.bytes(32).hex()


def servant_ip(i: int) -> str:
    return f"10.{(i >> 16) & 255}.{(i >> 8) & 255}.{i & 255}"


@dataclass
class Stream:
    name: str
    events: list
    meta: dict = field(default_factory=dict)


class Replayer:
    """Drives a TaskDispatcher with a Stream and records everything it returns."""

    def __init__(self, dispatcher: TaskDispatcher, *, pinned: bool = False, on_solve: Callable | None = None,
                 batch_heartbeats: bool = False, packed: bool = False, staged: bool = False, seed: int = 0):
        """`batch_heartbeats`: runs of consecutive "hb" events with one timestamp go through
        keep_servants_alive, runs of consecutive "notify"/"notify_own" events through
        notify_servants_running_tasks (one call each); the trace is the same by definition.

        `staged`: solves go through the device-side queue (yd_stage_requests + yd_wait_for_staged_tasks).  The trace is
        the same by definition.  Per solve, a generator seeded with `seed` picks how (`modes` records it):
          "exact"   stage the batch, decide it;
          "longer"  stage the batch followed by unrelated requests, decide the batch's prefix;
          "host"    the plain (or packed) call with the batch in a host array, which drops the staged queue (see
                    `_host_array` for how long the array lives);
          "reuse"   (not picked: taken whenever the batch is a prefix of what is still staged, e.g. the requests a
                    filtered call offered) decide it without staging again.
        Staged grants land in one grant array reused across calls."""
        self.d = dispatcher
        self.batch_heartbeats = batch_heartbeats
        self.packed = packed  # solves go through yd_wait_for_starting_new_tasks_packed (16-byte requests, 8-byte grants)
        self.pinned = pinned
        self.on_solve = on_solve
        self.staged = staged
        self.rng = np.random.default_rng(seed)
        self.modes: list[str] = []  # per solve call (staged mode), and "filter" per filtered call
        self.staged_q: np.ndarray | None = None  # host copy of the handle's staged queue, None once dropped
        self._host_bufs: list[np.ndarray] = []  # the host calls' request arrays, kept alive (see above)
        self._gout = np.zeros(0, dtype=GRANT_DTYPE)
        self.pending = np.zeros(0, dtype=REQ_DTYPE)
        self.outstanding: dict[int, int] = {}  # task id -> servant index at grant time
        self.decisions = 0
        self.granted = 0
        self.solve_calls = 0

    def _host_array(self, alloc: Callable, n: int) -> np.ndarray:
        """A page-locked request array for one host call.  Staged mode keeps every one alive until the replay ends and
        makes it at least 64 k requests long, so that a staged solve that read one of them instead of the device-side
        queue would read other requests, inside a live allocation."""
        if not self.staged:
            return alloc(n)
        self._host_bufs.append(alloc(max(n, 1 << 16)))
        return self._host_bufs[-1][:n]

    def _staged_mode(self, reqs: np.ndarray) -> str:
        n, q = len(reqs), self.staged_q
        if n and q is not None and len(q) >= n and (q[:n] == reqs).all():
            return "reuse"
        u = self.rng.random()
        return "host" if u < 0.2 else "longer" if u < 0.6 else "exact"

    def _wait(self, now: float, reqs: np.ndarray) -> np.ndarray:
        mode = self._staged_mode(reqs) if self.staged else "host"
        if self.staged:
            self.modes.append(mode)
        if mode != "host":
            n = len(reqs)
            if mode != "reuse":
                q = np.ascontiguousarray(reqs)
                if mode == "longer":  # unrelated requests behind the batch: the batch's own, rotated and reversed
                    tail = np.roll(q, int(self.rng.integers(1, max(n, 2))))[::-1][: int(self.rng.integers(1, max(n, 1) + 1))]
                    q = np.concatenate([q, tail])
                self.d.stage_requests(q)
                self.staged_q = q.copy()
            if len(self._gout) < n:
                self._gout = self.d.alloc_grants(2 * n) if self.pinned else np.zeros(2 * n, dtype=GRANT_DTYPE)
            g = self.d.wait_for_staged_tasks(n, now, out=self._gout).copy()
        elif self.packed:
            from .dispatcher import pack_requests
            if self.pinned:
                buf = pack_requests(reqs, self._host_array(self.d.alloc_requests16, len(reqs)))
                g = self.d.wait_for_starting_new_tasks_packed(buf, now, out8=self.d.alloc_grants8(len(reqs)))
            else:
                g = self.d.wait_for_starting_new_tasks_packed(pack_requests(reqs), now)
        elif self.pinned:
            buf = self._host_array(self.d.alloc_requests, len(reqs))
            buf[...] = reqs
            out = self.d.alloc_grants(len(reqs))
            g = self.d.wait_for_starting_new_tasks(buf, now, out=out).copy()
        else:
            g = self.d.wait_for_starting_new_tasks(np.ascontiguousarray(reqs), now).copy()
        if mode == "host" and len(reqs):
            self.staged_q = None
        self.decisions += len(reqs)
        ok = g["status"] == STATUS_GRANTED
        self.granted += int(ok.sum())
        self.solve_calls += 1
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        if self.on_solve:
            self.on_solve(self.d, reqs, g)
        return g

    def _filter(self, now: float, reqs: np.ndarray, cache_keys, task_digests) -> list[np.ndarray]:
        """One filtered call: [verdicts, in-flight hits, grants of the offered requests]."""
        reqs = np.ascontiguousarray(reqs)
        v, hits, g = self.d.filter_and_wait_for_starting_new_tasks(reqs, cache_keys, task_digests, now)
        g = g.copy()
        if len(reqs):  # the offered requests are the staged queue now (ydsched.h)
            self.staged_q = reqs[v == 0].copy()
        self.modes.append("filter")
        self.decisions += len(g)
        ok = g["status"] == STATUS_GRANTED
        self.granted += int(ok.sum())
        for tid, sidx in zip(g["task_id"][ok].tolist(), g["servant_index"][ok].tolist()):
            self.outstanding[tid] = sidx
        if self.on_solve:
            self.on_solve(self.d, reqs[v == 0], g)
        return [v.copy(), hits.copy(), g]

    def _notify_args(self, ev):
        """(location, tasks) of a notify / notify_own event, or None if the servant index is gone."""
        d = self.d
        if ev[0] == "notify":
            _, loc, tasks = ev
            return loc, [RunningTask(a, b, loc, c) for a, b, c in tasks]
        _, sidx, drop_seed, extra = ev
        loc = d.servant_location(sidx)
        if loc is None:
            return None
        own = sorted(t for t, s in self.outstanding.items() if s == sidx)
        rng = np.random.default_rng(drop_seed)
        own = [t for t in own if rng.random() < 0.8]
        ids = own + list(extra)
        return loc, [RunningTask(1000 + k, t, loc, f"{t:064x}") for k, t in enumerate(ids)]

    def run(self, stream: Stream) -> list[np.ndarray]:
        d = self.d
        trace: list[np.ndarray] = []
        events = stream.events
        pos = 0
        while pos < len(events):
            ev = events[pos]
            pos += 1
            kind = ev[0]
            if self.batch_heartbeats and kind == "hb":
                run = [ev]
                while pos < len(events) and events[pos][0] == "hb" and events[pos][1] == ev[1]:
                    run.append(events[pos])
                    pos += 1
                d.keep_servants_alive([e[2] for e in run], [e[3] for e in run], now=ev[1])
                continue
            if self.batch_heartbeats and kind in ("notify", "notify_own"):
                run = [ev]
                while pos < len(events) and events[pos][0] in ("notify", "notify_own"):
                    run.append(events[pos])
                    pos += 1
                # (servant indices and outstanding grants do not change inside the run: arguments up front)
                args = [self._notify_args(e) for e in run]
                res = iter(d.notify_servants_running_tasks([a for a in args if a is not None]))
                for a in args:
                    trace.append(np.asarray(next(res) if a is not None else [], dtype=np.uint64))
                continue
            if kind == "hb":
                _, now, sv, exp = ev
                d.keep_servant_alive(sv, exp, now=now)
            elif kind == "enqueue":
                self.pending = np.concatenate([self.pending, ev[1]])
            elif kind == "solve":
                g = self._wait(ev[1], self.pending)
                self.pending = self.pending[g["status"] == STATUS_TIMEOUT]
                trace.append(g)
            elif kind == "wait":
                trace.append(self._wait(ev[1], ev[2](d) if callable(ev[2]) else ev[2]))
            elif kind == "filter":
                trace += self._filter(*ev[1:])
            elif kind == "free":
                ids = np.asarray(ev[1], dtype=np.uint64)
                d.free_tasks(ids)
                for i in ids.tolist():
                    self.outstanding.pop(i, None)
            elif kind == "free_frac":
                _, seed, frac, *spare = ev
                ids = np.fromiter(sorted(self.outstanding), dtype=np.uint64, count=len(self.outstanding))
                rng = np.random.default_rng(seed)
                pick = ids[rng.random(len(ids)) < frac]
                if spare:
                    pick = pick[np.asarray([self.outstanding[i] not in spare[0] for i in pick.tolist()], dtype=bool)]
                d.free_tasks(pick)
                for i in pick.tolist():
                    self.outstanding.pop(i, None)
                trace.append(pick.copy())
            elif kind == "keepalive":
                _, now, ids, exp = ev
                if ids is None:
                    ids = sorted(self.outstanding)
                ok = d.keep_tasks_alive(np.asarray(ids, dtype=np.uint64), exp, now=now)
                trace.append(ok.astype(np.uint8))
            elif kind == "tick":
                d.on_expiration_timer(now=ev[1])
            elif kind == "notify":
                _, loc, tasks = ev
                unknown = d.notify_servant_running_tasks(
                    loc, [RunningTask(a, b, loc, c) for a, b, c in tasks]
                )
                trace.append(np.asarray(unknown, dtype=np.uint64))
            elif kind == "notify_own":
                _, sidx, drop_seed, extra = ev
                loc = d.servant_location(sidx)
                if loc is None:
                    trace.append(np.zeros(0, dtype=np.uint64))
                    continue
                own = sorted(t for t, s in self.outstanding.items() if s == sidx)
                rng = np.random.default_rng(drop_seed)
                own = [t for t in own if rng.random() < 0.8]
                ids = own + list(extra)
                unknown = d.notify_servant_running_tasks(
                    loc, [RunningTask(1000 + k, t, loc, f"{t:064x}") for k, t in enumerate(ids)]
                )
                trace.append(np.asarray(unknown, dtype=np.uint64))
            elif kind == "running":
                rt = d.get_running_tasks()
                trace.append(
                    np.asarray([(t.servant_task_id, t.task_grant_id) for t in rt], dtype=np.uint64).reshape(-1, 2)
                )
            elif kind == "state":
                st = d.servant_state()
                trace.append(
                    np.stack([st["running_tasks"], st["ever_assigned_tasks"], st["capacity_available"]], axis=1)
                    if len(st)
                    else np.zeros((0, 3), dtype=np.uint64)
                )
                trace.append(np.asarray([d.next_task_id(), d.num_tasks(), d.num_servants()], dtype=np.uint64))
            else:  # pragma: no cover
                raise ValueError(f"unknown event {kind!r}")
        return trace


def with_repeats(stream: Stream, seed: int, frac: float = 0.3) -> Stream:
    """The stream with, for a seeded `frac` of its "wait" batches, a prefix of that batch asked for again just before
    the next "wait" event (after whatever frees and ticks lie between).  A staged Replayer decides the repeat from the
    queue it staged for the first batch, without staging again."""
    rng = np.random.default_rng(seed)
    ev: list = []
    again = None
    for e in stream.events:
        if e[0] == "wait":
            if again is not None:
                ev.append(("wait", e[1], again))
            again = None
            if rng.random() < frac:
                part = float(rng.random())
                if callable(e[2]):  # (built again when the repeat runs: the same requests, the IPs already interned)
                    again = lambda dd, f=e[2], part=part: (lambda r: r[: max(1, int(len(r) * part))])(f(dd))  # noqa: E731
                elif len(e[2]):
                    again = e[2][: max(1, int(len(e[2]) * part))].copy()
        ev.append(e)
    return Stream(stream.name + "-repeats", ev, dict(stream.meta))


def trace_digest(trace: Sequence[np.ndarray]) -> str:
    h = hashlib.sha256()
    for a in trace:
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype.descr).encode())
        h.update(str(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def traces_equal(a: Sequence[np.ndarray], b: Sequence[np.ndarray]) -> bool:
    return len(a) == len(b) and all(x.shape == y.shape and x.dtype == y.dtype and (x == y).all() for x, y in zip(a, b))


def first_mismatch(a: Sequence[np.ndarray], b: Sequence[np.ndarray]) -> str:
    for k, (x, y) in enumerate(zip(a, b)):
        if x.shape != y.shape or x.dtype != y.dtype:
            return f"event-output {k}: shape/dtype {x.shape}/{x.dtype} vs {y.shape}/{y.dtype}"
        if not x.size:
            continue
        neq = np.nonzero(np.asarray(x != y).reshape(len(x), -1).any(axis=1))[0] if x.ndim else np.array([0])
        if (x != y).any():
            i = int(neq[0])
            return f"event-output {k}, row {i}: {x[i]!r} vs {y[i]!r} ({len(neq)} rows differ)"
    if len(a) != len(b):
        return f"trace lengths {len(a)} vs {len(b)}"
    return "equal"


# ---------------------------------------------------------------------------
# request / servant builders
# ---------------------------------------------------------------------------


def _requests(d: TaskDispatcher, env_ids: np.ndarray, ip_ids: np.ndarray, min_version, expires_in_s=15.0,
              prefetch=None) -> np.ndarray:
    r = np.zeros(len(env_ids), dtype=REQ_DTYPE)
    r["env_id"] = env_ids
    r["requestor_ip"] = ip_ids
    r["min_version"] = min_version
    r["expires_in_ns"] = int(expires_in_s * 1e9)
    if prefetch is not None:
        r["flags"] = np.where(prefetch, _abi.REQ_FLAG_PREFETCH, 0)
    return r


@dataclass
class Workload:
    """A config: servants to register and a function building its request queue."""

    name: str
    servants: list[Servant]
    digests: list[str]
    build_requests: Callable[[TaskDispatcher], np.ndarray]
    meta: dict = field(default_factory=dict)

    def register(self, d: TaskDispatcher, now: float = 0.0, expires_in: float = 10.0) -> None:
        for sv in self.servants:
            d.keep_servant_alive(sv, expires_in, now=now)

    def stream(self, d: TaskDispatcher) -> Stream:
        """Heartbeat x S, then one solve over the whole queue."""
        ev: list = [("hb", 0.0, sv, 10.0) for sv in self.servants]
        ev.append(("enqueue", self.build_requests(d)))
        ev.append(("solve", 0.001))
        ev.append(("state",))
        return Stream(self.name, ev, dict(self.meta))


def config1(n_tasks: int = 1000, n_servants: int = 64, seed: int = 42) -> Workload:
    """cfg 1: 1 k x 64, one digest held by everyone, uniform slots (SURVEY 8(d))."""
    rng = np.random.default_rng(seed)
    dg = hex_digest(rng)
    servants = [
        Servant(f"{servant_ip(i)}:8335", None, [dg], 8, 32, 0, 64 * GiB, 50 * GiB, 16, _abi.PRIORITY_USER)
        for i in range(n_servants)
    ]

    def build(d: TaskDispatcher) -> np.ndarray:
        e = d.intern_env(dg)
        ips = np.asarray([d.intern_ip(f"172.16.{i >> 8}.{i & 255}") for i in range(256)], dtype=np.uint32)
        r = np.random.default_rng(seed + 1)
        return _requests(d, np.full(n_tasks, e, np.uint32), ips[r.integers(0, 256, n_tasks)], 8)

    return Workload("cfg1", servants, [dg], build, {"tasks": n_tasks, "servants": n_servants, "digests": 1})


def config2(n_tasks: int = 100_000, n_servants: int = 2000, n_digests: int = 8, seed: int = 42,
            variant: str = "mod", max_tasks: int = 64, nproc: int = 128) -> Workload:
    """cfg 2: 100 k x 2 k, 8 digests, uniform slots; all grant.

    variant "mod":    servant i holds digest i mod 8  (8 independent components)
    variant "random": 1-3 random digests each         (one coupled component)
    """
    rng = np.random.default_rng(seed)
    dgs = [hex_digest(rng) for _ in range(n_digests)]
    servants = []
    for i in range(n_servants):
        if variant == "mod":
            envs = [dgs[i % n_digests]]
        else:
            k = int(rng.integers(1, 4))
            envs = [dgs[j] for j in rng.choice(n_digests, size=k, replace=False)]
        servants.append(
            Servant(f"{servant_ip(i)}:8335", None, envs, 8, nproc, 0, 256 * GiB, 200 * GiB, max_tasks, _abi.PRIORITY_USER)
        )

    def build(d: TaskDispatcher) -> np.ndarray:
        env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
        ips = np.asarray([d.intern_ip(f"172.16.{i >> 8}.{i & 255}") for i in range(4096)], dtype=np.uint32)
        r = np.random.default_rng(seed + 1)
        return _requests(d, env[r.integers(0, n_digests, n_tasks)], ips[r.integers(0, 4096, n_tasks)], 8)

    return Workload(f"cfg2-{variant}", servants, dgs, build,
                    {"tasks": n_tasks, "servants": n_servants, "digests": n_digests, "variant": variant})


def config3_task_sources(n: int = 100_000, seed: int = 47, n_tus: int = 6124, n_args: int = 40) -> "TaskSources":
    """The descriptors behind BASELINE configs[3]'s cache keys and task digests, for the 6124-TU trace looped to n
    requests: per TU a source digest (64 hex chars, as the delegate's BLAKE3 of the preprocessed source) and one of
    `n_args` invocation-argument strings whose lengths spread geometrically from about 100 B to 6 KiB, so that
    messages end inside the first chunk and several chunks in.  Request i is TU i mod n_tus."""
    from .dispatcher import TaskSources

    rng = np.random.default_rng(seed)
    words = ["-std=c++17", "-O2", "-g", "-fPIC", "-Wall", "-Wextra", "-DNDEBUG", "-fno-exceptions", "-pthread",
             "-fvisibility=hidden", "-ffunction-sections", "-fdata-sections", "-march=x86-64-v2", "-c", "-x", "c++"]
    args = []
    for length in np.geomspace(100, 6144, n_args).astype(int):
        parts: list[str] = []
        while sum(len(x) + 1 for x in parts) < length:
            parts.append(str(rng.choice(words)) if rng.random() < 0.6 else
                         f"-I/src/llvm/{rng.bytes(6).hex()}/include" if rng.random() < 0.7 else f"-D{rng.bytes(4).hex().upper()}=1")
        args.append(" ".join(parts)[:length])
    tu_args = rng.integers(0, n_args, n_tus).astype(np.uint32)
    tu_src = np.frombuffer(rng.bytes(32 * n_tus), dtype=np.uint8).reshape(n_tus, 32)
    hexd = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    tu_hex = np.stack([hexd[tu_src >> 4], hexd[tu_src & 15]], axis=2).reshape(n_tus, 64)
    tu = np.arange(n) % n_tus
    return TaskSources.of(args, tu_args[tu], np.ascontiguousarray(tu_hex[tu]))


def config_self(n_tasks: int = 100_000, n_servants: int = 2000, seed: int = 44, run_len: int = 4) -> Workload:
    """Production-like: ONE compiler digest, every requestor is itself a servant (so the
    self-exclusion rule, task_dispatcher.cc:372-379, is live for every request) and requests
    arrive in runs of `run_len` from the same machine (immediate_reqs > 1 per RPC)."""
    rng = np.random.default_rng(seed)
    dg = hex_digest(rng)
    servants = [
        Servant(f"{servant_ip(i)}:8335", None, [dg], 8, 128, int(rng.integers(0, 20)), 256 * GiB, 200 * GiB, 51,
                _abi.PRIORITY_DEDICATED if i % 10 == 0 else _abi.PRIORITY_USER)
        for i in range(n_servants)
    ]

    def build(d: TaskDispatcher) -> np.ndarray:
        e = d.intern_env(dg)
        ips = np.asarray([d.intern_ip(servant_ip(i)) for i in range(n_servants)], dtype=np.uint32)
        r = np.random.default_rng(seed + 1)
        who = np.repeat(r.integers(0, n_servants, (n_tasks + run_len - 1) // run_len), run_len)[:n_tasks]
        return _requests(d, np.full(n_tasks, e, np.uint32), ips[who], 8)

    return Workload("cfg-self", servants, [dg], build,
                    {"tasks": n_tasks, "servants": n_servants, "digests": 1, "self": "every requestor is a servant"})


def _mixed_servants(n_servants: int, dgs: list[str], rng: np.random.Generator, envs_per: str = "mod") -> list[Servant]:
    """cfg 3/5 servant mix: nproc in {32,64,96,128}; USER 40% / DEDICATED 95% capacity
    (daemon/cloud/execution_engine.cc:132,153); load ~ U[0,nproc]; 15% low memory;
    5% not accepting; versions {7,8}."""
    out = []
    for i in range(n_servants):
        nproc = int(rng.choice([32, 64, 96, 128]))
        dedicated = rng.random() < 0.10
        mt = nproc * 95 // 100 if dedicated else nproc * 40 // 100
        if rng.random() < 0.05:
            mt = 0
        load = int(rng.integers(0, nproc + 1))
        lowmem = rng.random() < 0.15
        total = 64 * GiB
        avail = int(rng.integers(1, 10)) * GiB - 1 if lowmem else int(rng.integers(11, 60)) * GiB
        ver = 7 if rng.random() < 0.3 else 8
        if envs_per == "mod":
            envs = [dgs[i % len(dgs)]]
        else:
            k = int(rng.integers(1, 4))
            envs = [dgs[j] for j in rng.choice(len(dgs), size=min(k, len(dgs)), replace=False)]
        out.append(
            Servant(f"{servant_ip(i)}:8335", None, envs, ver, nproc, load, total, avail, mt,
                    _abi.PRIORITY_DEDICATED if dedicated else _abi.PRIORITY_USER)
        )
    return out


def config3(n_tasks: int = 1_000_000, n_servants: int = 4000, n_digests: int = 8, seed: int = 43,
            envs_per: str = "random") -> Workload:
    """cfg 3: 1 M x 4 k, mixed memory headroom / priority / versions / self-IP.

    Capacity < tasks, so `rounds_stream` interleaves solves with Free and Tick.
    """
    rng = np.random.default_rng(seed)
    dgs = [hex_digest(rng) for _ in range(n_digests)]
    servants = _mixed_servants(n_servants, dgs, rng, envs_per)

    def build(d: TaskDispatcher) -> np.ndarray:
        env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
        r = np.random.default_rng(seed + 1)
        outside = np.asarray([d.intern_ip(f"172.16.{i >> 8}.{i & 255}") for i in range(4096)], dtype=np.uint32)
        inside = np.asarray([d.intern_ip(servant_ip(i)) for i in range(n_servants)], dtype=np.uint32)
        shares = r.random(n_tasks) < 0.20  # 20% of requestors are servants themselves
        ip = np.where(shares, inside[r.integers(0, n_servants, n_tasks)], outside[r.integers(0, 4096, n_tasks)])
        mv = np.where(r.random(n_tasks) < 0.5, 7, 8).astype(np.uint32)
        return _requests(d, env[r.integers(0, n_digests, n_tasks)], ip.astype(np.uint32), mv)

    return Workload("cfg3", servants, dgs, build,
                    {"tasks": n_tasks, "servants": n_servants, "digests": n_digests, "envs_per": envs_per})


def config5(n_tasks: int = 10_000_000, n_servants: int = 8000, n_digests: int = 8, seed: int = 45) -> Workload:
    w = config3(n_tasks, n_servants, n_digests, seed)
    return replace(w, name="cfg5")


def rounds_stream(w: Workload, d: TaskDispatcher, max_rounds: int = 8, free_frac: float = 0.5) -> Stream:
    """cfg 3 interleaving: solve, free a seeded half of the outstanding grants,
    renew the rest, re-heartbeat, tick +1 s, re-offer what is still pending."""
    ev: list = [("hb", 0.0, sv, 10.0) for sv in w.servants]
    ev.append(("enqueue", w.build_requests(d)))
    t = 0.001
    for k in range(max_rounds):
        ev.append(("solve", t))
        ev.append(("free_frac", 1000 + k, free_frac))
        ev.append(("keepalive", t + 0.5, None, 15.0))
        t += 1.0
        for sv in w.servants:
            ev.append(("hb", t, sv, 10.0))
        ev.append(("tick", t))
        ev.append(("state",))
    return Stream(w.name + "-rounds", ev, dict(w.meta, rounds=max_rounds))


# ---------------------------------------------------------------------------
# fuzz: every quirk at small scale
# ---------------------------------------------------------------------------


def fuzz_stream(d: TaskDispatcher, seed: int, n_servants: int = 24, n_events: int = 60, max_batch: int = 40,
                wide: bool = False, unique_hosts: bool = False) -> Stream:
    """Random interleaving of all event kinds over a small cluster.

    Covers: several ports on one IP (only the first free one is 'self'),
    requestors that are servants, dedicated servants around the 50% mark, low
    memory, max_tasks == 0, load above nproc, version gating incl. negative
    versions, unknown environments, capacity shrinking below running_tasks,
    lease expiry -> zombies -> sweep on heartbeat, servant expiry -> orphans,
    freeing unknown / duplicate ids, heartbeats from unknown locations.
    `wide` adds capacities above 32768 (the wide-key solver path).  `unique_hosts` gives every
    servant its own IP (one daemon per machine): requestors that are servants then have exactly
    one "self" servant, which is the shape the merge solver takes on itself.
    """
    rng = np.random.default_rng(seed)
    dgs = [hex_digest(rng) for _ in range(int(rng.integers(1, 5)))]
    hosts = [f"10.0.{i >> 8}.{i & 255}" for i in range(n_servants if unique_hosts else max(2, n_servants // 2))]

    def rand_servant(i: int) -> Servant:
        host = hosts[i] if unique_hosts else hosts[int(rng.integers(0, len(hosts)))]
        nproc = int(rng.choice([0, 2, 4, 8, 16, 32, 40000 if wide else 24]))
        mt = int(rng.choice([0, 2, 3, 7, 8, 12, 70000 if wide else 30]))
        k = int(rng.integers(0 if rng.random() < 0.2 else 1, len(dgs) + 1))
        envs = [dgs[j] for j in rng.choice(len(dgs), size=k, replace=False)] if k else []
        if rng.random() < 0.1:
            envs = envs + envs[:1]  # duplicate digest in one heartbeat
        return Servant(
            f"{host}:{8000 + i}",
            None,
            envs,
            int(rng.choice([-1, 6, 7, 8, 8, 9, 9])),
            nproc,
            int(rng.integers(0, max(nproc, 1) + 3)) if rng.random() < 0.4 else int(rng.integers(0, 3)),
            int(rng.choice([0, 64 * GiB])),
            int(rng.choice([5 * GiB, 10 * GiB - 1, 10 * GiB, 40 * GiB, 40 * GiB, 40 * GiB])),
            mt,
            int(rng.choice([_abi.PRIORITY_USER, _abi.PRIORITY_DEDICATED, _abi.PRIORITY_USER])),
        )

    servants = [rand_servant(i) for i in range(n_servants)]
    ev: list = []
    now = 0.0
    for sv in servants:
        ev.append(("hb", now, sv, float(rng.choice([2.0, 5.0, 10.0]))))
    env_ids = [d.intern_env(x) for x in dgs] + [d.intern_env("not-a-known-digest")]
    ip_pool = hosts + ["172.16.0.1", "172.16.0.2", "10.0.0", ""]
    ip_ids = [d.intern_ip(x) for x in ip_pool]
    issued = 0  # upper bound on ids handed out so far (for picking ids to free / renew)
    for _ in range(n_events):
        now += float(rng.choice([0.0, 0.1, 0.4, 1.0]))
        kind = rng.choice(["wait", "wait", "wait", "free", "keepalive", "tick", "hb", "notify", "running", "solve"])
        if kind in ("wait", "solve"):
            n = int(rng.integers(0, max_batch + 1))
            # runs of identical requests, like one RPC with immediate_reqs > 1
            e = np.repeat(rng.choice(env_ids, size=n), 1)
            ip = rng.choice(ip_ids, size=n)
            if n and rng.random() < 0.5:
                run = int(rng.integers(1, n + 1))
                e[:run] = e[0]
                ip[:run] = ip[0]
            r = _requests(d, e.astype(np.uint32), ip.astype(np.uint32),
                          rng.choice([0, 7, 8, 9], size=n).astype(np.uint32),
                          expires_in_s=float(rng.choice([0.5, 1.5, 15.0])), prefetch=rng.random(n) < 0.3)
            if kind == "wait":
                ev.append(("wait", now, r))
            else:
                ev.append(("enqueue", r))
                ev.append(("solve", now))
            issued += n
        elif kind == "free":
            k = int(rng.integers(0, 12))
            ids = rng.integers(0, issued + 3, size=k)
            if k and rng.random() < 0.3:
                ids[-1] = ids[0]  # duplicate
            ev.append(("free", ids.astype(np.uint64)))
        elif kind == "keepalive":
            k = int(rng.integers(0, 12))
            ev.append(("keepalive", now, rng.integers(0, issued + 3, size=k).astype(np.uint64),
                       float(rng.choice([0.5, 2.0, 15.0]))))
        elif kind == "tick":
            ev.append(("tick", now))
        elif kind == "hb":
            i = int(rng.integers(0, n_servants))
            if rng.random() < 0.5:
                servants[i] = replace(rand_servant(i), observed_location=servants[i].observed_location)
            ev.append(("hb", now, servants[i], float(rng.choice([0.0, 2.0, 5.0, 10.0]))))
        elif kind == "notify":
            if rng.random() < 0.15:
                ev.append(("notify", "203.0.113.9:1", [(1, int(rng.integers(0, issued + 3)), "aa")]))
            else:
                extra = rng.integers(0, issued + 3, size=int(rng.integers(0, 3))).tolist()
                ev.append(("notify_own", int(rng.integers(0, n_servants)), int(rng.integers(0, 1 << 30)), extra))
        elif kind == "running":
            ev.append(("running",))
        if rng.random() < 0.25:
            ev.append(("state",))
    ev.append(("state",))
    return Stream(f"fuzz-{seed}", ev, {"seed": seed, "servants": n_servants})


# ---------------------------------------------------------------------------
# solo: the one-launch solve's state from one call to the next
# ---------------------------------------------------------------------------

# What ends a steady stretch of `solo_stream`, and the path of the batch it bears on (fused.cuh, ydsched.cu WaitImpl):
#   hit        the speculative solve decides it on the kept class table and the kept slot order
#   rebuild    the speculative solve decides it, after the slot order was rebuilt
#   replay     the speculative solve misses; the batch is replayed on the clean scratch (variant 3)
#   standdown  the speculative solve misses; the replay stands down (flag 4) to the general sequence
#   fresh      a new topology: a full solo solve, no speculation
#   nospec     the batch cannot speculate
SOLO_MENU = {
    "version-up": "hit", "version-down": "hit", "version-drop-last": "hit",
    "load": "rebuild", "nproc": "rebuild", "max-tasks-0": "rebuild", "max-tasks-back": "rebuild",
    "low-memory": "rebuild", "priority": "rebuild",
    "keepalive": "hit", "free-unknown": "hit", "notify-bogus": "hit", "tick-leases": "hit", "tiny": "hit",
    "new-min-version": "replay", "new-digest": "replay",
    "self": "standdown", "two-min-versions": "standdown",
    "digest-set": "fresh", "new-servant": "fresh", "servant-expiry": "fresh",
    "size-class": "nospec", "class-bound": "nospec",
}
# perturbations that are a batch themselves (the others are events before the next stretch's first batch)
_SOLO_BATCHES = ("new-min-version", "new-digest", "self", "two-min-versions", "size-class", "class-bound")
_SIZE_CLASSES = {1024: (9, 1024), 2048: (1025, 2048), 4096: (2049, 3000)}  # Nb = NextPow2(n, 1024): n range


def _np2(x: int, lo: int) -> int:
    return max(lo, 1 << (max(x, 1) - 1).bit_length())


def solo_stream(d: TaskDispatcher, seed: int, *, wrap: bool | None = None, grow: bool | None = None) -> Stream:
    """Steady stretches of data-parallel batches (every servant holds one digest, one min_version per digest), each
    ended by one perturbation from SOLO_MENU, so that the one-launch solve's kept state -- slot order, class table,
    clean scratch, solo hint, servant facts on the device, lease ring -- is used and invalidated in every way a call
    sequence can.  meta["checks"] lists (batch, perturbation, expected path); a batch is the index of a "wait" event.

    `wrap` (default: every third seed): batches of 2049-3000 requests over a larger cluster, most grants freed after
    each, until more than 2^17 task ids were handed out -- the lease ring's live window crosses the ring's end.
    `grow` (default: every sixth seed): from about 20 000 ids on, the grants on servants 0 and 1 are neither freed
    nor swept, for 90 000 requests: the live window outgrows the ring while it straddles the ring's end.
    """
    rng = np.random.default_rng(seed)
    wrap = seed % 3 == 0 if wrap is None else wrap
    grow = seed % 6 == 0 if grow is None else grow
    K = 4 + seed % 9 if grow else 2 + seed % 11
    n_servants = int(rng.integers(400, 601)) if wrap else int(rng.integers(64, 301))
    dgs = [f"{0x50100000 + (seed << 8) + k:064x}" for k in range(K)]
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    unknown = np.asarray([d.intern_env(f"{0x5010dead + (seed << 8) + k:064x}") for k in range(2)], dtype=np.uint32)
    pins = (0, 1) if grow else ()
    net = 80 + seed % 100
    if seed % 4 == 1:  # shared hosts: three servants per IP, in three components (i mod K differ)
        host = lambda i: f"10.{net}.{(i // 3) >> 8}.{(i // 3) & 255}"  # noqa: E731
    else:
        host = lambda i: f"10.{net}.{i >> 8}.{i & 255}"  # noqa: E731

    def new_servant(i: int, digest: int) -> Servant:
        envs = [dgs[digest]] * (2 if rng.random() < 0.08 else 1)  # (a duplicate digest in one heartbeat)
        if i in pins:  # healthy, so that they hold grants from the first batch of the pinned window on
            return Servant(f"{host(i)}:{8000 + i}", None, envs, 9, 128, 0, 64 * GiB, 40 * GiB, 120, _abi.PRIORITY_USER)
        nproc = int(rng.choice([32, 64, 96, 128]))
        dedicated = rng.random() < 0.15
        if dedicated and rng.random() < 0.5:
            nproc += 1  # odd: the dedicated tier's edge 2r < P falls between two slots
        mt = nproc * 95 // 100 if dedicated else nproc * 40 // 100
        if rng.random() < 0.05:
            mt = 0
        if dedicated:
            load = nproc // 2 + int(rng.integers(-1, 2))
        elif rng.random() < 0.06:
            load = nproc + int(rng.integers(1, 8))  # load above nproc
        else:
            load = int(rng.integers(0, nproc + 1)) if rng.random() < 0.4 else int(rng.integers(0, 4))
        return Servant(f"{host(i)}:{8000 + i}", None, envs, int(rng.choice([-1, 6, 7, 8, 9, 9])), nproc, load,
                       64 * GiB, 5 * GiB if rng.random() < 0.15 else 40 * GiB, mt,
                       _abi.PRIORITY_DEDICATED if dedicated else _abi.PRIORITY_USER)

    # the registry as the scheduler keeps it, in position order (expired servants erased): (creation index, facts)
    sv: list[tuple[int, Servant]] = [(i, new_servant(i, i % K)) for i in range(n_servants)]
    made = n_servants
    ev: list = [("hb", 0.0, s, 1e6) for _, s in sv]
    # The id staging of FreeTask / KeepTaskAlive at its largest size first: a device buffer that grows drops the kept
    # class table (CleanSig holds the buffer generation), which would blur which event a path follows.
    bogus = np.arange(1 << 40, (1 << 40) + (1 << 17), dtype=np.uint64)
    ev += [("free", bogus), ("keepalive", 0.0, bogus, 1.0)]
    clients = np.asarray([d.intern_ip(f"172.30.{seed % 250}.{k}") for k in range(64)], dtype=np.uint32)
    late_names: list[str] = []  # client IPs that the batches intern themselves, after earlier solves
    zero = K - 1  # min_version 10, above every servant: EnvironmentNotFound with cls_nelig == 0
    mv = {k: int(rng.choice([7, 8, 9])) for k in range(K)}
    mv[zero] = 10
    classes = sorted({k for k in range(K - 1) if rng.random() < 0.7 or k < len(pins)} | {zero})
    if len(classes) == K and K > 2:
        classes.remove(K - 2)  # a held digest left out: the "new-digest" batch adds it
    size = 4096 if wrap else int(rng.choice(list(_SIZE_CLASSES)))
    st = {"now": 0.001, "issued": 0, "waits": 0, "pinned": False}
    checks: list = []
    saved_mt: list = []  # (location, max_tasks) of servants set to max_tasks 0
    dropped: list = []   # digests whose eligible servants all went below its min_version

    def digest_of(s: Servant) -> int:
        return dgs.index(s.environments[0])

    def holders(k: int) -> list[int]:
        return [p for p, (_, s) in enumerate(sv) if digest_of(s) == k]

    def movers() -> list[int]:  # positions whose servant may change or leave (pins stay as they are)
        return [p for p, (i, _) in enumerate(sv) if i not in pins]

    def pick(xs):
        return xs[int(rng.integers(0, len(xs)))]

    def hb(p: int, s: Servant, expires: float = 1e6) -> None:
        sv[p] = (sv[p][0], s)
        ev.append(("hb", st["now"], s, expires))

    def slot_b() -> int:
        return _np2(sum(min(s.num_processors, s.max_tasks) + 1 for _, s in sv), 4096)

    def between() -> None:  # after every batch: frees (not of the pinned grants), maybe a zombie sweep, a tick, state
        frac = 0.9 if wrap else 0.5
        ev.append(("free_frac", int(rng.integers(1 << 30)), frac) + ((pins,) if st["pinned"] else ()))
        if rng.random() < 0.3:
            ev.append(("notify_own", pick(movers()), int(rng.integers(1 << 30)), []))
        st["now"] += 0.003
        ev.append(("tick", st["now"]))
        ev.append(("state",))
        st["now"] += 0.003

    def batch(n: int, *, k=None, m=None, self_req: bool = False) -> None:
        """n requests over the stretch's digests (each at least once), 1 % unknown digests; requestors are clients,
        servants of other components, clients interned by this very batch, and (self_req) servants of their own."""
        if k is None:
            k = np.asarray(classes)[rng.integers(0, len(classes), n)]
            k[: min(n, len(classes))] = classes[: n]
        if m is None:
            m = np.asarray([mv[int(x)] for x in k], dtype=np.uint32)
        e = env[k]
        unk = rng.random(n) < 0.01
        unk[: len(classes) + 1] = False
        e[unk] = unknown[rng.integers(0, 2, int(unk.sum()))]
        by_host: dict[str, set[int]] = {}
        for _, s in sv:
            by_host.setdefault(s.observed_location.split(":")[0], set()).add(digest_of(s))
        names = sorted(by_host)
        hosts = {(c, o): [h for h in names if (c in by_host[h]) == o] for c in set(k.tolist()) for o in (False, True)}
        ips = clients[rng.integers(0, len(clients), n)]
        u = rng.random(n)
        own = (u < 0.1) if self_req else np.zeros(n, dtype=bool)
        own[0] = self_req
        for q in np.nonzero((u < 0.35) | own)[0].tolist():
            cand = hosts[int(k[q]), bool(own[q])]
            if cand:
                ips[q] = d.intern_ip(pick(cand))
        r = _requests(d, e, ips, m, expires_in_s=15.0, prefetch=rng.random(n) < 0.2)
        r["expires_in_ns"][rng.random(n) < 0.3] = 4_000_000  # short leases: zombies by the next tick
        late = np.nonzero((u > 0.93) & ~own)[0]
        if len(late):
            late_names.extend(f"192.168.{seed % 250}.{len(late_names) + j}" for j in range(int(rng.integers(1, 4))))
            names = [pick(late_names[-8:]) for _ in late]

            def build(dd, r=r, late=late, names=names):
                r = r.copy()
                r["requestor_ip"][late] = [dd.intern_ip(x) for x in names]
                return r
            ev.append(("wait", st["now"], build))
        else:
            ev.append(("wait", st["now"], r))
        st["waits"] += 1
        st["issued"] += n
        between()

    def stretch_n() -> int:
        lo, hi = _SIZE_CLASSES[size]
        return int(rng.integers(max(lo, K + 2), hi + 1))  # (room for every digest of the stretch)

    def facts(item: str) -> None:
        """One heartbeat that changes a slot fact or a flag but keeps slot_b (else: a new scratch layout)."""
        before = slot_b()
        for _ in range(200):
            p = pick(movers())
            s = sv[p][1]
            if item == "load":
                t = replace(s, current_load=int(rng.integers(0, s.num_processors + 4)))
            elif item == "nproc":
                t = replace(s, num_processors=int(rng.choice([32, 64, 96, 128, s.num_processors + 1])))
            elif item == "max-tasks-0":
                t = replace(s, max_tasks=0)
            elif item == "max-tasks-back":
                back = [(q, m0) for loc, m0 in saved_mt for q, (_, x) in enumerate(sv) if x.observed_location == loc]
                if back and rng.random() < 0.9:
                    p, m0 = back[0]
                    s = sv[p][1]
                    t = replace(s, max_tasks=m0)
                else:
                    t = replace(s, max_tasks=s.num_processors * 40 // 100 if s.max_tasks == 0 else s.max_tasks + 1)
            elif item == "low-memory":
                t = replace(s, memory_available_in_bytes=40 * GiB if s.memory_available_in_bytes < 10 * GiB else 5 * GiB)
            else:
                t = replace(s, priority=_abi.PRIORITY_USER if s.priority == _abi.PRIORITY_DEDICATED else
                            _abi.PRIORITY_DEDICATED)
            if t == s:
                continue
            sv[p] = (sv[p][0], t)
            if slot_b() == before:
                sv[p] = (sv[p][0], s)
                if item == "max-tasks-0":
                    saved_mt.append((s.observed_location, s.max_tasks))
                if item == "max-tasks-back":
                    saved_mt[:] = [x for x in saved_mt if x[0] != s.observed_location]
                hb(p, t)
                return
            sv[p] = (sv[p][0], s)
        raise AssertionError(f"solo_stream({seed}): no {item} heartbeat keeps slot_b")

    def perturb(item: str) -> None:
        nonlocal classes, made
        asked = [c for c in classes if c != zero]
        if item == "version-drop-last":  # every eligible servant of one asked-for digest below its min_version
            k = pick(asked or [zero])
            dropped.append(k)
            for p in holders(k):
                s = sv[p][1]
                if sv[p][0] not in pins and s.version >= mv[k]:
                    hb(p, replace(s, version=int(rng.choice([mv[k] - 1, -1]))))
        elif item == "version-up":  # those servants back up (else one servant)
            ps = holders(dropped.pop()) if dropped else [pick(movers())]
            for p in ps:
                if sv[p][0] not in pins:
                    hb(p, replace(sv[p][1], version=9))
        elif item == "version-down":  # one servant below its digest's min_version
            ps = [p for p in movers() if sv[p][1].version >= mv[digest_of(sv[p][1])]] or movers()
            p = pick(ps)
            hb(p, replace(sv[p][1], version=min(mv[digest_of(sv[p][1])], 9) - 1))
        elif item in ("load", "nproc", "max-tasks-0", "max-tasks-back", "low-memory", "priority"):
            facts(item)
        elif item == "keepalive":
            ev.append(("keepalive", st["now"], None, 15.0))
        elif item == "free-unknown":  # ids never handed out, one of them twice
            bogus = [st["issued"] + 10_000_000 + int(x) for x in rng.integers(0, 1000, 3)]
            ev.append(("free", np.asarray(bogus + bogus[:1], dtype=np.uint64)))
        elif item == "notify-bogus":
            ev.append(("notify_own", pick(movers()), int(rng.integers(1 << 30)),
                       [st["issued"] + 20_000_000, st["issued"] + 20_000_001]))
        elif item == "tick-leases":
            st["now"] += 0.02
            ev.append(("tick", st["now"]))
        elif item == "tiny":
            batch(int(rng.integers(1, 9)))
        elif item == "digest-set":  # the first holder of a digest, where it may move: the components are renumbered
            firsts = [holders(k)[0] for k in range(K) if holders(k)]
            ok = lambda p: sv[p][0] not in pins and len(holders(digest_of(sv[p][1]))) > 2  # noqa: E731
            p = pick([p for p in firsts if ok(p)] or [p for p in movers() if ok(p)])
            s = sv[p][1]
            k = (digest_of(s) + 1 + int(rng.integers(0, K - 1))) % K
            hb(p, replace(s, environments=[dgs[k]] * len(s.environments)))
        elif item == "new-servant":
            sv.append((made, new_servant(made, made % K)))
            made += 1
            ev.append(("hb", st["now"], sv[-1][1], 1e6))
        elif item == "servant-expiry":
            p = pick([p for p in movers() if len(holders(digest_of(sv[p][1]))) > 2])
            ev.append(("hb", st["now"], sv[p][1], 0.001))
            del sv[p]
            st["now"] += 0.002
            ev.append(("tick", st["now"]))
        elif item == "new-min-version" and asked:  # from this batch on
            k = pick(asked)
            mv[k] = int(rng.choice([x for x in (0, 6, 7, 8, 9) if x != mv[k]]))
            batch(stretch_n())
        elif item in ("new-digest", "new-min-version"):  # a held digest the table lacks, from this batch on
            missing = [k for k in range(K) if k not in classes and holders(k)]
            if missing:
                classes = sorted(classes + [missing[0]])
            else:  # every held digest is asked for: a new min_version instead
                k = pick(asked or [zero])
                mv[k] = int(rng.choice([x for x in (0, 6, 7, 8, 9) if x != mv[k]]))
            batch(stretch_n())
        elif item == "self":
            batch(stretch_n(), self_req=True)
        elif item == "two-min-versions":
            n = stretch_n()
            k = np.asarray(classes)[rng.integers(0, len(classes), n)]
            k[: len(classes)] = classes
            m = np.asarray([mv[int(x)] for x in k], dtype=np.uint32)
            two = pick(asked or [zero])
            other = mv[two] - 1 if 0 < mv[two] <= 9 else 1
            m[(k == two) & (rng.random(n) < 0.5)] = other
            m[len(classes)] = other
            k[len(classes)] = two
            batch(n, k=k, m=m)
        elif item == "size-class":
            lo, hi = _SIZE_CLASSES[int(rng.choice([c for c in _SIZE_CLASSES if c != size]))]
            batch(int(rng.integers(lo, hi + 1)))
        elif item == "class-bound":  # every digest at enough min_versions for 40+ classes: the bound grows
            per = -(-40 // K)  # (a "self" batch may have taken it from 16 to 32 already)
            n = max(stretch_n(), K * per)
            k = rng.integers(0, K, n)
            m = rng.integers(0, per, n).astype(np.uint32)
            k[: K * per] = np.repeat(np.arange(K), per)
            m[: K * per] = np.tile(np.arange(per, dtype=np.uint32), K)
            batch(n, k=k, m=m)
        else:  # pragma: no cover
            raise KeyError(item)

    order = list(SOLO_MENU)
    rng.shuffle(order)
    target = 3 << 16 if wrap else 0  # requests offered: enough that the task ids handed out pass 2^17
    passes = 0
    while True:
        passes += 1
        for item in order:
            if grow and st["issued"] >= 20_000 and "pin_from" not in st:
                ev.append(("free_frac", int(rng.integers(1 << 30)), 1.0))  # the pinned window starts here
                st["pin_from"], st["pinned"] = st["issued"], True
            elif st["pinned"] and st["issued"] - st["pin_from"] >= 90_000:
                st["pinned"] = False
                ev.append(("free_frac", int(rng.integers(1 << 30)), 1.0))  # the pinned grants go
            for _ in range(int(rng.integers(3, 5))):  # a steady stretch
                batch(stretch_n())
            if st["pinned"]:
                ev.append(("keepalive", st["now"], None, 15.0))
            at = st["waits"]
            perturb(item)
            checks.append((at if item in _SOLO_BATCHES else st["waits"], item, SOLO_MENU[item]))
        if st["issued"] >= target and not st["pinned"]:
            break
        order = [x for x in SOLO_MENU if x != "class-bound"]  # (the bound has grown; it stays)
        rng.shuffle(order)
    for _ in range(3):
        batch(stretch_n())
    ev.append(("state",))
    return Stream(f"solo-{seed}", ev, {"seed": seed, "servants": n_servants, "digests": K, "wrap": wrap, "grow": grow,
                                       "checks": checks, "waits": st["waits"], "passes": passes})


# ---------------------------------------------------------------------------
# named streams (used by tests/golden and the parity tests)
# ---------------------------------------------------------------------------


def named_stream(name: str, d: TaskDispatcher) -> Stream:
    """Deterministic stream by name; the same names are keys in
    tests/golden/digests.json."""
    if name == "cfg1":
        return config1().stream(d)
    if name == "cfg2-mod-small":
        return config2(5000, 200, 8, variant="mod").stream(d)
    if name == "cfg2-random-small":
        return config2(5000, 200, 8, variant="random").stream(d)
    if name == "cfg2-mod":
        return config2(variant="mod").stream(d)
    if name == "cfg2-random":
        return config2(variant="random").stream(d)
    if name == "cfg-self-small":
        return config_self(6000, 150).stream(d)
    if name == "cfg-self":
        return config_self().stream(d)
    if name == "cfg3-small":
        return rounds_stream(config3(20000, 300, 8), d, max_rounds=4)
    if name == "cfg3-mod-small":
        return rounds_stream(config3(20000, 300, 8, envs_per="mod"), d, max_rounds=4)
    if name == "cfg3":
        return rounds_stream(config3(), d, max_rounds=3)
    if name == "cfg5-1m":  # BASELINE configs[4]'s servant pool and distributions, first 1 M requests of its queue
        return config5(1_000_000, 8000).stream(d)
    if name == "cfg5-1m-rounds":
        return rounds_stream(config5(1_000_000, 8000), d, max_rounds=2)
    if name.startswith("fuzz-"):
        seed = int(name.split("-")[1])
        return fuzz_stream(d, seed, n_servants=8 + seed % 30, wide=(seed % 5 == 0))
    raise KeyError(name)
