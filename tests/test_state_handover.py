"""State export / import (include/ydstate.h): a handle imported from an export makes the same decisions,
call after call, as the handle that never stopped.

CPU cases run the port's state build (checkers/libydport_state.so) and compare with the verbatim
reference run that never stopped; GPU cases compare the CUDA backend's exports byte for byte with the
port's and continue CUDA handles imported from either backend."""
import os
import signal
import socket
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

from conftest import REF_LIB, ROOT
from solve_lines import solves
from yadcc_b200 import _abi
from yadcc_b200 import streams as S
from yadcc_b200.dispatcher import RunningTask, Servant, StateError, TaskDispatcher, _ns

PORT_STATE_LIB = ROOT / "checkers" / "libydport_state.so"
FUZZ_SEEDS = list(range(24))
SMALL_STREAMS = ["cfg1", "cfg2-mod-small", "cfg-self-small", "cfg3-small"]


@pytest.fixture(scope="session")
def state_lib():
    if not PORT_STATE_LIB.exists():
        subprocess.check_call(["make", "-C", str(ROOT), "checkers/libydport_state.so"])
    return str(PORT_STATE_LIB)


# ---- the format, read independently of the C codec --------------------------------------------


def parse(blob: bytes) -> dict:
    """Decode an export as ydstate.h documents it; records where each section starts."""
    at = 0
    off = {}

    def get(fmt):
        nonlocal at
        v = struct.unpack_from("<" + fmt, blob, at)
        at += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def string():
        nonlocal at
        n = get("I")
        s = blob[at:at + n].decode()
        at += n
        return s

    h = dict(zip(("magic", "version", "id_stride", "id_offset", "min_mem", "next_task_id"), get("IIIIQQ")))
    off["envs"] = at
    h["envs"] = [string() for _ in range(get("I"))]
    off["ips"] = at
    h["ips"] = [string() for _ in range(get("I"))]
    h["servants"] = []
    for _ in range(get("I")):
        f = dict(zip(("version", "priority", "reason", "nproc", "load", "max_tasks", "total_mem", "avail_mem",
                      "expires_rel", "ever"), get("iiiIIIQQqQ")))
        f["observed"], f["reported"] = string(), string()
        f["envs"] = [string() for _ in range(get("I"))]
        h["servants"].append(f)
    off["leases"] = at
    n = get("Q")
    h["leases"] = np.frombuffer(blob, dtype=[("id", "<u8"), ("servant", "<u4"), ("flags", "<u4"), ("rel", "<i8")],
                                count=n, offset=at).copy()
    at += 24 * n
    off["bookkeeper"] = at
    h["bucket_count"] = get("Q")
    h["groups"] = []
    for _ in range(get("I")):
        loc = string()
        h["groups"].append((loc, [(get("Q"), get("Q"), string(), string()) for _ in range(get("I"))]))
    assert at == len(blob)
    h["_off"] = off
    return h


# ---- driving a stream with cuts -----------------------------------------------------------------


def _event_time(ev):
    return ev[1] if ev[0] in ("hb", "solve", "wait", "keepalive", "tick", "filter") else None


def cut_points(stream: S.Stream, k: int = 6) -> list[int]:
    n = len(stream.events)
    return sorted({max(1, n * i // (k + 1)) for i in range(1, k + 1)} - {n})


def pre_intern(d: TaskDispatcher, stream: S.Stream) -> None:
    """Intern every digest servants report and every servant IP prefix the CUDA backend interns on its own, so that
    the intern tables of all backends fed this stream are the same (ydstate.h)."""
    for ev in stream.events:
        if ev[0] == "hb":
            sv: Servant = ev[2]
            for e in sv.environments:
                d.intern_env(e)
            loc = sv.observed_location
            for k, c in enumerate(loc):
                if c == ":":
                    d.intern_ip(loc[:k])


def run_cut(make, name: str, cuts, *, handover: bool, intern: bool = False):
    """Replay stream `name`, exporting at every cut; with `handover` each export goes into a fresh handle from
    `make(i)` (i = the segment's number) that plays the rest.  Returns (trace, exports, final handle)."""
    d = make(0)
    stream = S.named_stream(name, d)
    if intern:
        pre_intern(d, stream)
    rp = S.Replayer(d)
    trace, exports, now, start = [], [], 0.0, 0
    for i, c in enumerate(list(cuts) + [len(stream.events)]):
        seg = stream.events[start:c]
        trace += rp.run(S.Stream(name, seg))
        for ev in seg:
            t = _event_time(ev)
            now = t if t is not None else now
        start = c
        if c == len(stream.events):
            break
        blob = d.export_state(now=now)
        exports.append(blob)
        if handover:
            d = make(i + 1)
            d.import_state(blob, now=now)
            rp.d = d
    trace.append(final_answers(d))
    return trace, exports, d


def final_answers(d: TaskDispatcher) -> np.ndarray:
    """What the handle answers at the end: servant state (expiry included), running tasks in order, next id."""
    st = d.servant_state()
    rt = d.get_running_tasks()
    parts = [st["running_tasks"], st["ever_assigned_tasks"], st["capacity_available"], st["expires_at_ns"].astype(np.uint64),
             np.asarray([(t.servant_task_id, t.task_grant_id) for t in rt], dtype=np.uint64).ravel(),
             np.asarray([d.next_task_id(), d.num_tasks(), d.num_servants()], dtype=np.uint64)]
    return np.concatenate([np.asarray(p, dtype=np.uint64) for p in parts])


def _lib_factory(lib):
    made = []

    def make(_i):
        made.append(TaskDispatcher(lib))
        return made[-1]

    return make, made


def _close(*lists):
    for ds in lists:
        for d in ds:
            d.close()


# ---- the reference's side of an export --------------------------------------------------------------------------
# The verbatim reference has no export; what an export must hold is read from the reference itself: servants, their
# personalities, expiry and counters, next_task_id and GetRunningTasks through its C ABI, the intern tables from the
# ids it handed out, and the leases (not observable through the ABI) from a model fed every call the reference gets.


class ReferenceLeases(TaskDispatcher):
    """A dispatcher over the reference library that also keeps the lease map as TaskDispatcher (task_dispatcher.cc)
    changes it: grants (:123-135), FreeTask (:167-188), KeepTaskAlive (:142-165), the zombie sweep of a heartbeat
    (:453-476), and the timer's servant drop, orphan sweep and zombie marking (:498-536)."""

    def __init__(self, lib):
        super().__init__(lib)
        self.leases: dict[int, list] = {}  # id -> [servant location, expires_at_ns, prefetch, zombie]
        self.groups: set[str] = set()      # RunningTaskBookkeeper's keys

    def _locations(self):
        return [self.servant_location(i) for i in range(self.num_servants())]

    def wait_for_starting_new_tasks(self, reqs, now=0.0, *, now_ns=None, out=None):
        t = now_ns if now_ns is not None else _ns(now)
        g = super().wait_for_starting_new_tasks(reqs, now, now_ns=now_ns, out=out)
        self._granted(t, reqs, g)
        return g

    def filter_and_wait_for_starting_new_tasks(self, reqs, cache_keys=None, task_digests=None, now=0.0, **kw):
        v, hits, g = super().filter_and_wait_for_starting_new_tasks(reqs, cache_keys, task_digests, now, **kw)
        self._granted(_ns(now), reqs[v == 0], g)
        return v, hits, g

    def _granted(self, now_ns, reqs, g):
        locs = self._locations()
        for r, x in zip(reqs, g):
            if x["status"] == _abi.STATUS_GRANTED:
                self.leases[int(x["task_id"])] = [locs[int(x["servant_index"])], now_ns + int(r["expires_in_ns"]),
                                                  bool(r["flags"] & _abi.REQ_FLAG_PREFETCH), False]

    def free_tasks(self, task_ids):
        ids = [int(i) for i in task_ids]
        super().free_tasks(ids)
        for i in ids:
            self.leases.pop(i, None)

    def keep_tasks_alive(self, task_ids, new_expires_in, *, now=0.0):
        ids = [int(i) for i in task_ids]
        ok = super().keep_tasks_alive(ids, new_expires_in, now=now)
        for i, k in zip(ids, ok):
            if k:
                self.leases[i][1] = _ns(now) + _ns(new_expires_in)
        return ok

    def notify_servant_running_tasks(self, servant_location, tasks):
        if servant_location in self._locations():
            reported = {t.task_grant_id for t in tasks}
            for i in [i for i, x in self.leases.items() if x[0] == servant_location and x[3] and i not in reported]:
                del self.leases[i]
            self.groups.add(servant_location)
        return super().notify_servant_running_tasks(servant_location, tasks)

    def notify_servants_running_tasks(self, batch):
        return [self.notify_servant_running_tasks(loc, tasks) for loc, tasks in batch]

    def on_expiration_timer(self, *, now):
        t = _ns(now)
        st = self.servant_state()
        gone = {loc for loc, e in zip(self._locations(), st["expires_at_ns"].tolist()) if e < t}
        super().on_expiration_timer(now=now)
        self.groups -= gone
        self.leases = {i: x for i, x in self.leases.items() if x[0] not in gone}
        for x in self.leases.values():
            x[3] = x[3] or x[1] < t

    def expected_export(self, now: float) -> dict:
        """Every field of the export the reference determines; the bookkeeper as GetRunningTasks shows it."""
        t = _ns(now)
        assert len(self.leases) == self.num_tasks()  # the model holds what the reference holds
        envs = sorted(self._env_ids.items(), key=lambda kv: kv[1])
        ips = sorted(self._ip_ids.items(), key=lambda kv: kv[1])
        assert [v for _, v in envs] == list(range(len(envs)))
        locs = self._locations()
        st = self.servant_state()
        servants = []
        for i in range(len(locs)):
            p = self.servant_personality(i)
            servants.append(dict(version=p.version, priority=p.priority, reason=p.not_accepting_task_reason,
                                 nproc=p.num_processors, load=p.current_load, max_tasks=p.max_tasks,
                                 total_mem=p.total_memory_in_bytes, avail_mem=p.memory_available_in_bytes,
                                 expires_rel=int(st["expires_at_ns"][i]) - t, ever=int(st["ever_assigned_tasks"][i]),
                                 observed=p.observed_location, reported=p.reported_location, envs=list(p.environments)))
        pos = {loc: i for i, loc in enumerate(locs)}
        leases = [(i, pos[x[0]], (1 if x[2] else 0) | (2 if x[3] else 0), x[1] - t) for i, x in sorted(self.leases.items())]
        return dict(next_task_id=self.next_task_id(), min_mem=self.parse_size("10G"), envs=[k for k, _ in envs],
                    ips=[""] + [k for k, v in ips if v != 0], servants=servants, leases=leases, groups=set(self.groups),
                    running=[(x.servant_task_id, x.task_grant_id, x.servant_location, x.task_digest)
                             for x in self.get_running_tasks()])


def assert_export_matches_reference(blob: bytes, want: dict, what: str = "") -> None:
    h = parse(blob)
    assert (h["magic"], h["version"], h["id_stride"], h["id_offset"]) == (0x54534459, 1, 1, 0), what
    for k in ("next_task_id", "min_mem", "envs", "ips", "servants"):
        assert h[k] == want[k], f"{what}: {k}"
    got = [tuple(int(v) for v in r) for r in h["leases"].tolist()]
    assert got == want["leases"], f"{what}: leases"
    # the groups, in the bookkeeper's iteration order: GetRunningTasks lists them last-iterated first
    assert {loc for loc, _ in h["groups"]} == want["groups"], f"{what}: bookkeeper keys"
    assert [t for _, tasks in reversed(h["groups"]) for t in tasks] == want["running"], f"{what}: bookkeeper order"


def reference_exports(name: str, cuts) -> tuple[list, list[dict]]:
    """The reference run that never stops: its trace, and at every cut what the export must hold."""
    if not REF_LIB.exists():
        pytest.skip("oracle/_ref/libydref.so not built (needs the reference sources)")
    ref = ReferenceLeases(str(REF_LIB))
    stream = S.named_stream(name, ref)
    rp = S.Replayer(ref)
    trace, wants, now, start = [], [], 0.0, 0
    for c in list(cuts) + [len(stream.events)]:
        seg = stream.events[start:c]
        trace += rp.run(S.Stream(name, seg))
        for ev in seg:
            t = _event_time(ev)
            now = t if t is not None else now
        start = c
        if c != len(stream.events):
            wants.append(ref.expected_export(now))
    trace.append(final_answers(ref))
    ref.close()
    return trace, wants


# ---- CPU: port chains against the reference that never stopped ----------------------------------


@pytest.mark.parametrize("name", [f"fuzz-{s}" for s in FUZZ_SEEDS] + SMALL_STREAMS)
def test_port_handover_matches_uninterrupted_reference(name, state_lib):
    d0 = TaskDispatcher(state_lib)
    cuts = cut_points(S.named_stream(name, d0))
    d0.close()
    ref_trace, wants = reference_exports(name, cuts)
    make, made = _lib_factory(state_lib)
    try:
        plain, plain_exports, _ = run_cut(make, name, cuts, handover=False)
        chain, chain_exports, _ = run_cut(make, name, cuts, handover=True)  # port -> port -> ... at every cut
    finally:
        _close(made)
    assert S.traces_equal(plain, ref_trace), S.first_mismatch(plain, ref_trace)
    assert S.traces_equal(chain, ref_trace), S.first_mismatch(chain, ref_trace)
    # at every cut the export holds what the reference holds ...
    for i, (blob, want) in enumerate(zip(plain_exports, wants)):
        assert_export_matches_reference(blob, want, f"cut {i}")
    # ... and it is canonical: the handed-over handles export what the one that never stopped exports
    assert chain_exports == plain_exports


def test_golden_cases_round_trip(state_lib):
    """The reference's own test scenarios: the export holds what the reference holds at the end, and the imported
    handle answers like the reference handle that ran the scenario and exports the same bytes."""
    from golden_cases import ALL_CASES

    if not REF_LIB.exists():
        pytest.skip("oracle/_ref/libydref.so not built (needs the reference sources)")
    for case in ALL_CASES:
        a = TaskDispatcher(state_lib)
        ref = ReferenceLeases(str(REF_LIB))
        try:
            case(a)
            case(ref)
            blob = a.export_state(now=1000.0)
            assert_export_matches_reference(blob, ref.expected_export(1000.0), case.__name__)
            b = TaskDispatcher(state_lib)
            b.import_state(blob, now=1000.0)
            assert b.export_state(now=1000.0) == blob, case.__name__
            ra, rb = final_answers(ref), final_answers(b)
            assert ra.shape == rb.shape and (ra == rb).all(), case.__name__
            b.close()
        finally:
            a.close()
            ref.close()


def test_service_streams_handover(state_lib, make_dispatcher):
    """The service layer (token checks, RPC expansion) over a handed-over dispatcher answers like the uninterrupted
    reference: heartbeats, grants, renewals and frees continue across the cut."""
    from yadcc_b200.service import HeartbeatRequest, SchedulerService

    def scenario(make, cut):
        d = make()
        outs = []
        for step in range(40):
            if step == cut:
                blob = d.export_state(now=step)
                d = make()
                d.import_state(blob, now=step)
            svc = SchedulerService(d, acceptable_user_tokens="u", acceptable_servant_tokens="s", now=0.0)
            rng = np.random.default_rng(step)
            for k in range(int(rng.integers(1, 4))):
                loc = f"10.0.0.{k + 1}:{8000 + k}"
                own = [t for t in outs[-1:] for t in t] if outs else []
                r = svc.heartbeat(HeartbeatRequest(token="s", location=loc, remote_ip=f"10.0.0.{k + 1}", version=9,
                                                   num_processors=8, capacity=int(rng.integers(1, 6)), servant_priority=2,
                                                   env_digests=["d" * 64],
                                                   running_tasks=[RunningTask(1, t, loc, f"{t:064x}") for t in own[k::3]]),
                                  now=step)
                outs.append([r.status] + sorted(r.expired_tasks))
            rpcs = np.zeros(2, dtype=_abi.RPC_WAIT_DTYPE)
            rpcs["env_id"] = d.intern_env("d" * 64)
            rpcs["requestor_ip"] = d.intern_ip("10.9.9.9")
            rpcs["immediate_reqs"] = rng.integers(0, 4, 2)
            rpcs["prefetch_reqs"] = rng.integers(0, 2, 2)
            rpcs["next_keep_alive_ns"] = 5_000_000_000
            res, g = svc.wait_for_starting_tasks(["u", "u"], rpcs, now=step)
            outs.append(res["status"].tolist() + g["task_id"].tolist())
            st, ok = svc.keep_task_alive("u", g["task_id"][::2], 3000, now=step)
            outs.append([st] + ok.tolist())
            svc.free_task("u", g["task_id"][1::3])
            if step % 3 == 2:
                d.on_expiration_timer(now=step + 0.5)
            outs.append([t.task_grant_id for t in d.get_running_tasks()] + [d.next_task_id()])
            svc.close()
        return outs

    ref = scenario(lambda: make_dispatcher("ref"), cut=None)
    made = []
    for cut in (5, 17, 31):
        got = scenario(lambda: made.append(TaskDispatcher(state_lib)) or made[-1], cut=cut)
        assert got == ref, cut
    _close(made)


def _small_blob(lib, **kw) -> tuple[bytes, TaskDispatcher]:
    """A handle with servants, leases (a zombie and a prefetch among them) and bookkeeping, and its export."""
    d = TaskDispatcher(lib, **kw)
    for k in range(3):
        d.keep_servant_alive(Servant(f"10.0.0.{k}:80", environments=["e" * 64, "f" * 64], version=3, num_processors=4,
                                     max_tasks=3, priority=1 + k % 2), 30, now=0)
    r = d.make_requests(6, "e" * 64, "10.0.0.1", expires_in=2)
    r["flags"][::2] = _abi.REQ_FLAG_PREFETCH
    g = d.wait_for_starting_new_tasks(r, now=1)
    d.make_requests(1, "f" * 64, "10.0.0.9")
    d.keep_tasks_alive(g["task_id"][1:], 20, now=2)
    d.on_expiration_timer(now=4)  # the first grant becomes a zombie
    for k in range(3):
        loc = f"10.0.0.{k}:80"
        mine = [int(t) for t, s in zip(g["task_id"], g["servant_index"]) if s == k]
        d.notify_servant_running_tasks(loc, [RunningTask(7, t, loc, f"{t:064x}") for t in mine])
    d.free_task(int(g["task_id"][-1]))
    return d.export_state(now=5), d


def test_format_fields(state_lib):
    blob, d = _small_blob(state_lib)
    h = parse(blob)
    assert h["next_task_id"] == d.next_task_id() == 6 and h["min_mem"] == 10 << 30
    assert h["ips"][0] == "" and h["envs"] == ["e" * 64, "f" * 64]
    assert [s["observed"] for s in h["servants"]] == [d.servant_location(i) for i in range(3)]
    assert h["leases"]["id"].tolist() == [0, 1, 2, 3, 4]
    assert h["leases"]["flags"].tolist() == [3, 0, 1, 0, 1]  # zombie | prefetch, then the renewed ones
    assert h["leases"]["rel"].tolist() == [-2 * 10**9] + [17 * 10**9] * 4
    st = d.servant_state()
    assert [s["ever"] for s in h["servants"]] == st["ever_assigned_tasks"].tolist()
    assert [s["expires_rel"] for s in h["servants"]] == [25 * 10**9] * 3
    assert len(h["groups"]) == 3
    d.close()


def test_import_rebases_time(state_lib):
    """Time stands still while the state is in transit: a lease with 10 s left at export has 10 s left after import."""
    a = TaskDispatcher(state_lib)
    a.keep_servant_alive(Servant("10.0.0.1:80", environments=["e" * 64], num_processors=4, max_tasks=4), 30, now=0)
    g = a.wait_for_starting_new_tasks(a.make_requests(2, "e" * 64, "10.0.0.2", expires_in=15), now=5)
    b = TaskDispatcher(state_lib)
    b.import_state(a.export_state(now=10), now=5000)
    assert b.servant_state()["expires_at_ns"].tolist() == [5020 * 10**9]
    b.on_expiration_timer(now=5009.5)
    assert b.keep_tasks_alive([int(g["task_id"][0])], 15, now=5009.5).all()  # renewed: now expires at 5024.5
    b.on_expiration_timer(now=5010.5)  # the other one expired at 5010: a zombie now
    assert b.keep_tasks_alive(g["task_id"].tolist(), 15, now=5010.5).tolist() == [True, False]
    assert b.next_task_id() == 2 and b.num_tasks() == 2
    a.close()
    b.close()


def test_import_refusals(state_lib):
    blob, a = _small_blob(state_lib)
    used = TaskDispatcher(state_lib)
    used.intern_env("x")
    with pytest.raises(StateError) as e:
        used.import_state(blob)
    assert e.value.code == _abi.STATE_NOT_FRESH
    done = TaskDispatcher(state_lib)
    done.import_state(blob)
    with pytest.raises(StateError) as e:
        done.import_state(blob)  # an imported handle is not fresh either
    assert e.value.code == _abi.STATE_NOT_FRESH
    for kw in ({"servant_min_memory_for_accepting_new_task": "1G"}, {"id_stride": 2, "id_offset": 0}):
        other = TaskDispatcher(state_lib, **kw)
        with pytest.raises(StateError) as e:
            other.import_state(blob)
        assert e.value.code == _abi.STATE_CONFIG_MISMATCH
        other.close()
    for x in (a, used, done):
        x.close()


def test_strided_ids_round_trip(state_lib):
    blob, a = _small_blob(state_lib, id_stride=4, id_offset=3)
    h = parse(blob)
    assert (h["id_stride"], h["id_offset"], h["next_task_id"]) == (4, 3, 27)
    assert (h["leases"]["id"] % 4 == 3).all()
    b = TaskDispatcher(state_lib, id_stride=4, id_offset=3)
    b.import_state(blob, now=5)
    assert b.export_state(now=5) == blob
    g = b.wait_for_starting_new_tasks(b.make_requests(1, "e" * 64, "10.0.0.9"), now=6)
    assert g["task_id"].tolist() == [27]
    a.close()
    b.close()


def corruptions(blob: bytes) -> dict[str, bytes]:
    """One corrupted export per rule of ydstate.h's input checks."""
    h = parse(blob)
    lo = h["_off"]["leases"]
    rec = lo + 8  # first lease record

    def put(fmt, at, v, b=blob):
        b = bytearray(b)
        struct.pack_into("<" + fmt, b, at, v)
        return bytes(b)

    n = len(h["leases"])
    out = {
        "magic": put("I", 0, 0x12345678),
        "version": put("I", 4, 2),
        "zero stride": put("I", 8, 0),
        "offset >= stride": put("I", 12, 1),
        "next id not ours": put("Q", 24, h["next_task_id"] + 1, put("I", 8, 2)),
        "env count overruns": put("I", h["_off"]["envs"], 1 << 30),
        "ip count overruns": put("I", h["_off"]["ips"], 1 << 30),
        "string length overruns": put("I", h["_off"]["envs"] + 4, len(blob)),
        "lease count overruns": put("Q", lo, n + 1000),
        "lease servant out of range": put("I", rec + 8, len(h["servants"])),
        "lease ids unsorted": put("Q", rec + 24, 0, put("Q", rec, 1)),
        "lease ids duplicated": put("Q", rec + 24, h["leases"]["id"][0]),
        "lease id at next_task_id": put("Q", rec + 24 * (n - 1), h["next_task_id"]),
        "lease id not congruent": put("Q", rec + 24 * (n - 1), h["leases"]["id"][-1] + 1, put("I", 8, 2)),
        "lease flags unknown": put("I", rec + 12, 8),
        "bucket count zero": put("Q", h["_off"]["bookkeeper"], 0),
        "bucket count absurd": put("Q", h["_off"]["bookkeeper"], 1 << 40),
        "group count overruns": put("I", h["_off"]["bookkeeper"] + 8, 1 << 20),
        "running-task count overruns": put("I", h["_off"]["bookkeeper"] + 12 + 4 + len(h["groups"][0][0]), 1 << 28),
        "trailing byte": blob + b"\0",
        "live window wider than 2^40 ids": put("Q", 24, int(h["leases"]["id"][0]) + (1 << 40) + 1),
        "next id near 2^64": put("Q", 24, (1 << 64) - 1),
        "next id with its top bit flipped": put("Q", 24, h["next_task_id"] | (1 << 63)),
        "ip 0 not empty": put("I", h["_off"]["ips"] + 4, 1) [: h["_off"]["ips"] + 8] + b"x" + blob[h["_off"]["ips"] + 8:],
    }
    return out


def check_malformed(lib: str) -> int:
    """Every truncation and every corruption is refused with BAD_BLOB and leaves the handle fresh."""
    blob, a = _small_blob(lib)
    a.close()
    d = TaskDispatcher(lib)
    checked = 0
    for k in range(len(blob)):
        with pytest.raises(StateError) as e:
            d.import_state(blob[:k])
        assert e.value.code == _abi.STATE_BAD_BLOB, k
        checked += 1
    for what, bad in corruptions(blob).items():
        with pytest.raises(StateError) as e:
            d.import_state(bad)
        assert e.value.code == _abi.STATE_BAD_BLOB, what
        checked += 1
    d.import_state(blob, now=5)  # still fresh after all that
    assert d.export_state(now=5) == blob
    d.close()
    return checked


def test_malformed_input_is_refused(state_lib):
    assert check_malformed(state_lib) > 100


@pytest.mark.gpu
def test_malformed_input_is_refused_by_cuda(cuda_lib):
    """The CUDA import refuses the same inputs without touching the device, and stays fresh; a valid export whose live
    window cannot fit the device (2^39 ids: a 16 TiB ring) is refused as such, not as malformed."""
    assert check_malformed(cuda_lib) > 100
    blob, a = _small_blob(cuda_lib)
    a.close()
    wide = bytearray(blob)
    struct.pack_into("<Q", wide, 24, int(parse(blob)["leases"]["id"][0]) + (1 << 39))
    d = TaskDispatcher(cuda_lib)
    with pytest.raises(StateError) as e:
        d.import_state(bytes(wide), now=5)
    assert e.value.code == _abi.STATE_NO_MEMORY
    d.import_state(blob, now=5)
    assert d.export_state(now=5) == blob
    d.close()


def test_malformed_input_under_asan(tmp_path):
    """The same checks against an AddressSanitizer build of the port's state library."""
    gxx = "g++"
    asan = subprocess.run([gxx, "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.isabs(asan):
        pytest.skip("no libasan for this compiler")
    lib = tmp_path / "libydport_state_asan.so"
    subprocess.check_call([gxx, "-std=gnu++2a", "-O1", "-g", "-fPIC", "-fsanitize=address", "-fno-omit-frame-pointer",
                           "-w", f"-I{ROOT / 'include'}", "-shared", "-o", str(lib), str(ROOT / "checkers" / "port_state.cc")])
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_state_handover as T\n"
            "print('checked', T.check_malformed(%r))\n") % (str(ROOT / "tests"), str(ROOT), str(lib))
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0:exitcode=23")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=str(ROOT / "tests"),
                       timeout=600)
    assert r.returncode == 0 and "checked" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_bookkeeper_order_survives_growth(state_lib, make_dispatcher):
    """GetRunningTasks' order (the bookkeeper map's iteration order) after import, and after later inserts push the map
    past its bucket count, against the reference that never stopped."""
    rng = np.random.default_rng(7)
    plan = []
    for step in range(300):
        k = int(rng.integers(0, 120 if step < 150 else 400))
        plan.append(("hb", k, step))
        if rng.random() < 0.05:
            plan.append(("tick", None, step + 0.5))

    def play(d, events, expiry):
        for kind, k, t in events:
            if kind == "tick":
                d.on_expiration_timer(now=t)
                continue
            loc, dg = f"10.1.{k // 256}.{k % 256}:80", f"{k:064x}"
            d.keep_servant_alive(Servant(loc, environments=[dg], num_processors=1000, max_tasks=1000), expiry(k), now=t)
            # a fresh grant on this servant (its digest is its own), reported at once: every group holds one task
            a = d.wait_for_starting_new_task("1.1.1.1", 0, dg, 100, now=t)
            d.notify_servant_running_tasks(loc, [RunningTask(k, a.task_id, loc, dg)] if hasattr(a, "task_id") else [])

    expiry = lambda k: 3 if k % 7 == 0 else 1000  # noqa: E731
    ref = make_dispatcher("ref")
    play(ref, plan, expiry)
    want = [t.servant_location for t in ref.get_running_tasks()]
    got_all = []
    for cut in (40, 150, 220):
        a = TaskDispatcher(state_lib)
        play(a, plan[:cut], expiry)
        t = max(e[2] for e in plan[:cut])
        b = TaskDispatcher(state_lib)
        b.import_state(a.export_state(now=t), now=t)
        play(b, plan[cut:], expiry)
        got_all.append([x.servant_location for x in b.get_running_tasks()])
        a.close()
        b.close()
    assert len(want) > 50 and all(g == want for g in got_all)
    ref2 = make_dispatcher("ref")
    outs = []
    for d in (ref2, TaskDispatcher(state_lib)):
        play(d, plan[:150], expiry)
        if d.backend != "reference":
            c = TaskDispatcher(state_lib)
            c.import_state(d.export_state(now=149), now=149)
            d.close()
            d = c
        for k in range(400, 900):  # far past the bucket count the cut saw
            loc = f"10.2.{k // 256}.{k % 256}:80"
            d.keep_servant_alive(Servant(loc, environments=["e" * 64], num_processors=2, max_tasks=2), 1000, now=150)
            d.notify_servant_running_tasks(loc, [RunningTask(k, 0, loc, "x")])
        outs.append([(t.servant_task_id, t.servant_location) for t in d.get_running_tasks()])
        if d.backend != "reference":
            d.close()
    assert outs[0] == outs[1]


# ---- the server: stop with --state, restart --------------------------------------------------------


def test_scheduler_server_restart_keeps_leases(tmp_path, state_lib):
    pytest.importorskip("google.protobuf")
    import asyncio

    sys.path.insert(0, str(ROOT / "tools"))
    import wire_protos as W

    PB = W.PB
    state = tmp_path / "sched.state"

    def start():
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        p = subprocess.Popen([sys.executable, str(ROOT / "tools" / "scheduler_server.py"), "--port", str(port),
                              "--user-tokens", "usr", "--servant-tokens", "srv", "--library", state_lib, "--window-ms", "2",
                              "--state", str(state)], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        for _ in range(200):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.1).close()
                return p, port
            except OSError:
                time.sleep(0.05)
        p.kill()
        raise RuntimeError(p.communicate()[1].decode())

    async def rpc(port, method, msg, resp):
        r, w = await asyncio.open_connection("127.0.0.1", port)
        w.write(W.request_frame(method, msg, 1))
        await w.drain()
        hdr = await r.readexactly(16)
        _, ms, bs, att = struct.unpack("<IIII", hdr)
        out = W.parse_response_frame(hdr + await r.readexactly(ms + bs + att), resp)
        w.close()
        return out

    def heartbeat(port, running=()):
        hb = PB["HeartbeatRequest"](token="srv", next_heartbeat_in_ms=10000, version=9, location="127.0.0.1:9000",
                                    num_processors=8, capacity=4, servant_priority=2)
        hb.env_descs.add().compiler_digest = "c" * 64
        for t in running:
            hb.running_tasks.add(servant_task_id=1, task_grant_id=t, servant_location="127.0.0.1:9000",
                                 task_digest="a" * 64)
        meta, body = asyncio.run(rpc(port, "Heartbeat", hb, PB["HeartbeatResponse"]))
        assert meta.response_meta.status == 0
        return list(body.expired_tasks)

    def grant(port, n):
        wq = PB["WaitForStartingTaskRequest"](token="usr", immediate_reqs=n, next_keep_alive_in_ms=10000)
        wq.env_desc.compiler_digest = "c" * 64
        meta, body = asyncio.run(rpc(port, "WaitForStartingTask", wq, PB["WaitForStartingTaskResponse"]))
        assert meta.response_meta.status == 0
        return [g.task_grant_id for g in body.grants]

    p, port = start()
    try:
        heartbeat(port)
        ids = grant(port, 2)
        assert ids == [0, 1]
    finally:
        p.send_signal(signal.SIGTERM)
        assert p.wait(timeout=30) == 0, p.stderr.read().decode()
    assert state.exists() and parse(state.read_bytes())["next_task_id"] == 2
    p, port = start()
    try:
        ka = PB["KeepTaskAliveRequest"](token="usr", next_keep_alive_in_ms=10000)
        ka.task_grant_ids.extend(ids)
        meta, body = asyncio.run(rpc(port, "KeepTaskAlive", ka, PB["KeepTaskAliveResponse"]))
        assert list(body.statuses) == [True, True]
        assert heartbeat(port, running=ids) == []  # the servant is not told to kill anything
        assert grant(port, 1) == [2]  # ids continue where the old process stopped
    finally:
        p.send_signal(signal.SIGINT)
        assert p.wait(timeout=30) == 0, p.stderr.read().decode()


# ---- GPU ------------------------------------------------------------------------------------------------------


GPU_STREAMS = [f"fuzz-{s}" for s in FUZZ_SEEDS] + SMALL_STREAMS


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_STREAMS)
def test_cuda_exports_match_port(name, state_lib, cuda_lib):
    """At every cut the CUDA export is the port's, byte for byte; CUDA handles imported from CUDA exports, and from
    port exports, continue exactly like the port."""
    d0 = TaskDispatcher(state_lib)
    cuts = cut_points(S.named_stream(name, d0))
    d0.close()
    made = []

    def maker(kinds):
        def make(i):
            made.append(TaskDispatcher(state_lib if kinds[i % len(kinds)] == "port" else cuda_lib))
            return made[-1]
        return make

    try:
        port_trace, port_exports, _ = run_cut(maker(["port"]), name, cuts, handover=False, intern=True)
        cuda_trace, cuda_exports, _ = run_cut(maker(["cuda"]), name, cuts, handover=False, intern=True)
        chain_trace, chain_exports, _ = run_cut(maker(["cuda"]), name, cuts, handover=True, intern=True)
        mixed_trace, mixed_exports, _ = run_cut(maker(["cuda", "port"]), name, cuts, handover=True, intern=True)
    finally:
        _close(made)
    for i, (a, b) in enumerate(zip(port_exports, cuda_exports)):
        assert a == b, f"cut {i}: {describe_difference(a, b)}"
    assert chain_exports == port_exports and mixed_exports == port_exports
    for t in (cuda_trace, chain_trace, mixed_trace):
        assert S.traces_equal(port_trace, t), S.first_mismatch(port_trace, t)


def describe_difference(a: bytes, b: bytes) -> str:
    ha, hb = parse(a), parse(b)
    for k in ("next_task_id", "envs", "ips", "bucket_count", "groups"):
        if ha[k] != hb[k]:
            return f"{k} differs"
    if ha["servants"] != hb["servants"]:
        return "servants differ"
    la, lb = ha["leases"], hb["leases"]
    if len(la) != len(lb) or not (la == lb).all():
        return f"leases differ ({len(la)} vs {len(lb)})"
    return "?"


def _solo_cut_run(lib_first, lib_rest, seed, cuts_every):
    """solo_stream (solo / coupled / self-request batches, ring wrap and growth, churn) cut every `cuts_every` events."""
    d = TaskDispatcher(lib_first)
    stream = S.solo_stream(d, seed, wrap=True, grow=True)
    pre_intern(d, stream)
    cuts = list(range(cuts_every, len(stream.events), cuts_every))
    rp = S.Replayer(d)
    trace, exports, now, start, handles = [], [], 0.0, 0, [d]
    for c in cuts + [len(stream.events)]:
        seg = stream.events[start:c]
        trace += rp.run(S.Stream("solo", seg))
        for ev in seg:
            t = _event_time(ev)
            now = t if t is not None else now
        start = c
        if c == len(stream.events):
            break
        blob = d.export_state(now=now)
        exports.append(blob)
        if lib_rest is not None:
            d = TaskDispatcher(lib_rest)
            d.import_state(blob, now=now)
            handles.append(d)
            rp.d = d
    trace.append(final_answers(d))
    _close(handles)
    return trace, exports


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_cuda_solo_stream_handover(seed, state_lib, cuda_lib):
    p_trace, p_exports = _solo_cut_run(state_lib, None, seed, 25)
    c_trace, c_exports = _solo_cut_run(cuda_lib, None, seed, 25)
    h_trace, h_exports = _solo_cut_run(cuda_lib, cuda_lib, seed, 25)
    assert c_exports == p_exports and h_exports == p_exports
    assert any(len(parse(b)["leases"]) and (parse(b)["leases"]["flags"] & 2).any() for b in p_exports), "no zombie was carried"
    for t in (c_trace, h_trace):
        assert S.traces_equal(p_trace, t), S.first_mismatch(p_trace, t)


GPU_CHILD = r"""
import sys, os
sys.path[:0] = [{tests!r}, {root!r}]
import numpy as np
from yadcc_b200 import TaskDispatcher, streams as S
from yadcc_b200.dispatcher import Servant
a = TaskDispatcher({lib!r})
servants = [Servant(f"10.3.{{k // 256}}.{{k % 256}}:80", environments=["e" * 64], num_processors=64, max_tasks=64, priority=2)
            for k in range(256)]
a.keep_servants_alive(servants, 1e6, now=0)
r = a.make_requests(2048, "e" * 64, "10.9.9.9", expires_in=60)
for t in range(3):
    g = a.wait_for_starting_new_tasks(r, now=1 + t)
    a.free_tasks(g["task_id"][g["status"] == 2])
b = TaskDispatcher({lib!r})
b.import_state(a.export_state(now=4), now=4)
print("IMPORTED", flush=True)
for t in range(5):
    g = b.wait_for_starting_new_tasks(r, now=5 + t)
    b.free_tasks(g["task_id"][g["status"] == 2])
"""


@pytest.mark.gpu
def test_cuda_import_returns_to_speculative_solve(cuda_lib, tmp_path):
    """After import, the first solo batch rebuilds the kept class table and steady-state solo batches run the
    speculative solve again (variant 4 on the YDSCHED_DEBUG line)."""
    code = GPU_CHILD.format(tests=str(ROOT / "tests"), root=str(ROOT), lib=cuda_lib)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, YDSCHED_DEBUG="1"))
    assert r.returncode == 0, r.stderr[-3000:]
    lines = solves(r.stderr)
    assert len(lines) == 8, r.stderr[-3000:]
    pre, post = [s.get("variant") for s in lines[:3]], [s.get("variant") for s in lines[3:]]
    assert pre[2] == 4, pre  # the handle that never stopped speculates from its third solo batch
    assert post[0] != 4 and post[2:] == [4] * 3, post  # imported: cold first, then speculative again


@pytest.mark.gpu
def test_cuda_handover_at_configs2_scale(cuda_lib):
    """BASELINE configs[2] (cfg3: 1 M requests over 4 k servants): cut right after the first solve, when the most
    leases are live, continue on an imported handle; the trace digest is the uninterrupted run's stored reference
    digest."""
    import json

    name = "cfg3"
    golden = json.loads((ROOT / "tests" / "golden" / "digests.json").read_text())["streams"][name]["sha256"]
    d = TaskDispatcher(cuda_lib)
    stream = S.named_stream(name, d)
    rp = S.Replayer(d, pinned=True)
    cut = next(i for i, ev in enumerate(stream.events) if ev[0] == "solve") + 1
    trace = rp.run(S.Stream(name, stream.events[:cut]))
    now = max(t for t in map(_event_time, stream.events[:cut]) if t is not None)
    t0 = time.perf_counter()
    blob = d.export_state(now=now)
    t1 = time.perf_counter()
    e = TaskDispatcher(cuda_lib)
    e.import_state(blob, now=now)
    t2 = time.perf_counter()
    leases = len(parse(blob)["leases"])
    assert e.export_state(now=now) == blob
    d.close()
    rp.d = e
    trace += rp.run(S.Stream(name, stream.events[cut:]))
    e.close()
    print(f"{name}: {leases} live leases at the cut, export {1e3 * (t1 - t0):.1f} ms, import {1e3 * (t2 - t1):.1f} ms")
    assert leases >= 100_000  # (every grant of the first solve: the servants' free capacity bounds it)
    assert S.trace_digest(trace) == golden, "handed-over run differs from the stored reference digest"


def _million_lease_stream(d):
    """4 k servants with 256 free slots each; one solve of 1 M requests fills them all, then frees, a tick and more
    solves churn the leases."""
    servants = [Servant(f"{S.servant_ip(k)}:8335", environments=["e" * 64], num_processors=256, max_tasks=256,
                        priority=1 + k % 2) for k in range(4000)]
    ev = [("hb", 0.0, sv, 1e6) for sv in servants]
    r = d.make_requests(1_000_000, "e" * 64, "172.16.0.1", expires_in=30)
    ev += [("wait", 1.0, r), ("state",), ("free_frac", 1, 0.4), ("tick", 2.0), ("wait", 3.0, r[:500_000]),
           ("free_frac", 2, 0.3), ("tick", 40.0), ("wait", 41.0, r[:300_000]), ("state",)]
    return ev


MILLION_DIGESTS = ROOT / "tests" / "golden" / "state_handover_digests.json"


def million_lease_reference_digest(lib) -> str:
    """Trace digest of the uninterrupted run of _million_lease_stream (what tests/golden/state_handover_digests.json
    stores, made with the reference library: `python tests/test_state_handover.py oracle/_ref/libydref.so`)."""
    d = TaskDispatcher(lib)
    trace = S.Replayer(d).run(S.Stream("1m", _million_lease_stream(d))) + [final_answers(d)]
    d.close()
    return S.trace_digest(trace)


@pytest.mark.gpu
def test_cuda_handover_with_a_million_live_leases(cuda_lib):
    """About 1 M live leases over 4 k servants, cut right after the solve that made them: the handed-over run's trace
    is the stored digest of the verbatim reference's uninterrupted run, and the handed-over handle exports what the
    handle that never stopped exports at the next cut."""
    import json

    golden = json.loads(MILLION_DIGESTS.read_text())["1m-leases"]["sha256"]
    traces, exports = [], []
    for handover in (False, True):
        d = TaskDispatcher(cuda_lib)
        ev = _million_lease_stream(d)
        rp = S.Replayer(d, pinned=True)
        trace = rp.run(S.Stream("1m", ev[:4001]))
        blob = d.export_state(now=1.0)
        if handover:
            e = TaskDispatcher(cuda_lib)
            e.import_state(blob, now=1.0)
            d.close()
            d = rp.d = e
        trace += rp.run(S.Stream("1m", ev[4001:]))
        exports.append((blob, d.export_state(now=41.0)))
        traces.append(trace + [final_answers(d)])
        d.close()
    assert len(parse(exports[0][0])["leases"]) == 1_000_000
    assert exports[0] == exports[1]
    assert S.traces_equal(traces[0], traces[1]), S.first_mismatch(traces[0], traces[1])
    assert S.trace_digest(traces[1]) == golden, "handed-over run differs from the reference's stored digest"


if __name__ == "__main__":
    print(million_lease_reference_digest(sys.argv[1]))
