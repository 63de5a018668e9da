"""Runs of Heartbeat, KeepTaskAlive and FreeTask frames (yd_wire_handle_frames batches each run into one service call),
checked against the same frames through yd_wire_call one by one.

`Twins` drives two services fed the same windows: `a` gets each window as one yd_wire_handle_frames call, `b` every
frame through yd_wire_call in order.  Every frame's status, error description and response body must be byte-equal,
and after every window so must the dispatchers' state (servant state, next task id, lease count, running tasks and,
where the library exports it, the whole decision state of ydstate.h).  `random_window` builds seeded windows: runs of
1 to 64 same-method frames mixed with WaitForStartingTask windows, GetConfig, GetRunningTasks, frames answered early,
ticks and token roll-outs.  The targeted cases each pin one rule of the batched handlers.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

from yadcc_b200.service import SchedulerService

import wire_protos as W

PB = W.PB
ENVS = [f"{i:02x}" * 32 for i in range(3)]
GIB = 1 << 30
USER, SERVANT, ROLLOUT_S, MIN_VERSION = "u1,u2", "s1,u2", 3, 2
IPS = [f"10.7.0.{k}" for k in range(10)] + ["172.16.0.1", "172.16.0.9"]


@dataclass
class Frame:
    method: str  # short name; "Nope" is answered early (unknown method)
    body: bytes
    ip: str


def hb_frame(k: int, *, token="s1", ip=None, location=None, ms=5000, version=3, running=(), capacity=4) -> Frame:
    ip = ip if ip is not None else f"10.7.0.{k}"
    m = PB["HeartbeatRequest"](token=token, next_heartbeat_in_ms=ms, version=version,
                               location=location if location is not None else f"10.7.0.{k}:8335", num_processors=16,
                               current_load=1, servant_priority=2, capacity=capacity, total_memory_in_bytes=64 * GIB,
                               memory_available_in_bytes=50 * GIB)
    for e in ENVS[: 1 + k % 3]:
        m.env_descs.add().compiler_digest = e
    for j, t in enumerate(running):
        r = m.running_tasks.add()
        r.servant_task_id, r.task_grant_id, r.servant_location, r.task_digest = 40 + j, int(t), m.location, f"{int(t):064x}"
    return Frame("Heartbeat", m.SerializeToString(), ip)


def wait_frame(*, token="u1", env=0, imm=2, pre=0, ka_ms=10000, ip="172.16.0.1") -> Frame:
    m = PB["WaitForStartingTaskRequest"](token=token, immediate_reqs=imm, prefetch_reqs=pre, next_keep_alive_in_ms=ka_ms)
    m.env_desc.compiler_digest = ENVS[env]
    return Frame("WaitForStartingTask", m.SerializeToString(), ip)


def keep_frame(ids, *, token="u1", ms=10000) -> Frame:
    m = PB["KeepTaskAliveRequest"](token=token, next_keep_alive_in_ms=ms)
    m.task_grant_ids.extend(int(x) for x in ids)
    return Frame("KeepTaskAlive", m.SerializeToString(), "172.16.0.2")


def free_frame(ids, *, token="u1") -> Frame:
    m = PB["FreeTaskRequest"](token=token)
    m.task_grant_ids.extend(int(x) for x in ids)
    return Frame("FreeTask", m.SerializeToString(), "172.16.0.3")


def config_frame(token="u1") -> Frame:
    return Frame("GetConfig", PB["GetConfigRequest"](token=token).SerializeToString(), "172.16.0.4")


def running_frame() -> Frame:
    return Frame("GetRunningTasks", b"", "172.16.0.4")


def unknown_frame() -> Frame:
    return Frame("Nope", b"", "172.16.0.5")


def _parse(frame: bytes):
    """(status, description, body) of a response frame."""
    ms = struct.unpack("<I", frame[4:8])[0]
    meta = PB["RpcMeta"]()
    meta.ParseFromString(frame[16:16 + ms])
    return meta.response_meta.status, meta.response_meta.description, frame[16 + ms:]


class Mismatch(AssertionError):
    pass


class Twins:
    def __init__(self, make_a, make_b, *, seed=5):
        mk = lambda d: SchedulerService(d, acceptable_user_tokens=USER, acceptable_servant_tokens=SERVANT,  # noqa: E731
                                        min_daemon_version=MIN_VERSION, serving_daemon_token_rollout_interval=ROLLOUT_S,
                                        token_seed=seed, now=0.0)
        self.a, self.b = mk(make_a()), mk(make_b())
        # The intern tables are part of the exported state, and a run of WaitForStartingTask frames interns its
        # requestors before its solve: every address and environment of the streams is interned up front.
        for d in (self.a.dispatcher, self.b.dispatcher):
            for ip in IPS:
                d.intern_ip(ip)
            for e in ENVS:
                d.intern_env(e)
        self.corr = 0
        self.windows = 0

    def close(self):
        self.a.close()
        self.b.close()

    def window(self, frames: list[Frame], now: float):
        """One window: `a` through yd_wire_handle_frames, `b` frame by frame through yd_wire_call.  Returns b's
        answers [(status, description, body)]."""
        wire = []
        for f in frames:
            self.corr += 1
            wire.append((_frame(f, self.corr), f.ip))
        outs = self.a.handle_frames(wire, now=now)
        answers = []
        for k, (f, o) in enumerate(zip(frames, outs)):
            st, desc, body = self.b.call(W.SERVICE + f.method, f.body, f.ip, now=now)
            got = _parse(o[3])
            want = (st, desc if st else "", body if st == 0 else b"")
            if o[0] != 1 or got != want:
                raise Mismatch(f"window {self.windows} frame {k} ({f.method}): frames {got!r} != calls {want!r}")
            answers.append(want)
        self.compare(now)
        self.windows += 1
        return answers

    def tick(self, now: float):
        self.a.dispatcher.on_expiration_timer(now=now)
        self.b.dispatcher.on_expiration_timer(now=now)
        self.compare(now)

    def compare(self, now: float):
        da, db = self.a.dispatcher, self.b.dispatcher
        checks = [("servant state", lambda d: d.servant_state().tobytes()), ("next task id", lambda d: d.next_task_id()),
                  ("lease count", lambda d: d.num_tasks()), ("running tasks", lambda d: d.get_running_tasks())]
        # (the exported bytes also hold intern tables, whose order is each library's own: compared within one library)
        if exports_state(da) and exports_state(db) and da._lib._name == db._lib._name:
            checks.append(("exported state", lambda d: d.export_state(now=now)))
        for what, f in checks:
            if f(da) != f(db):
                raise Mismatch(f"after window {self.windows}: {what} differs")


def exports_state(d) -> bool:
    return hasattr(d._lib, "yd_export_state")


def _frame(f: Frame, corr: int) -> bytes:
    meta = PB["RpcMeta"](correlation_id=corr, method_type=1)
    meta.request_meta.method_name = W.SERVICE + f.method
    mb = meta.SerializeToString()
    return struct.pack("<IIII", W.MAGIC, len(mb), len(f.body), 0) + mb + f.body


# ---- seeded streams ------------------------------------------------------------------------------------------------------
RUN_LENGTHS = [1, 1, 2, 3, 5, 8, 16, 33, 64]


def _ids(rng, next_id: int, n: int):
    top = next_id + 4
    out = [int(x) for x in rng.integers(0, max(top, 1), size=n)]
    if n and rng.random() < 0.3:
        out[int(rng.integers(0, n))] = 10**12 + int(rng.integers(0, 9))  # far outside the window
    if n > 1 and rng.random() < 0.4:
        out[-1] = out[0]  # a duplicate
    return out


def _random_hb(rng, next_id: int) -> Frame:
    k = int(rng.integers(0, 10))
    kind = rng.random()
    kw = dict(token=str(rng.choice(["s1", "s1", "s1", "u1", "u2", "bad"])), ms=int(rng.choice([0, 1000, 5000, 5000, 30000, 30001])),
              version=int(rng.choice([1, 3, 3, 3])), capacity=int(rng.choice([0, 2, 4, 8])))
    if kind < 0.15:  # behind NAT: reports servant k's location from another servant's address
        kw["ip"] = f"10.7.0.{int(rng.integers(0, 10))}"
    elif kind < 0.2:
        kw["location"] = str(rng.choice(["nonsense", "10.7.0.1:99999", "[::1]:8335"]))
    if next_id and rng.random() < 0.7:
        kw["running"] = _ids(rng, next_id, int(rng.integers(0, 8)))
    return hb_frame(k, **kw)


def random_window(rng, next_id: int) -> list[Frame]:
    frames: list[Frame] = []
    for _ in range(int(rng.integers(1, 5))):
        m = str(rng.choice(["hb", "hb", "keep", "free", "wait", "config", "running"]))
        n = int(rng.choice(RUN_LENGTHS))
        for i in range(n if m in ("hb", "keep", "free") else int(rng.integers(1, 4)) if m == "wait" else 1):
            if rng.random() < 0.04:
                frames.append(unknown_frame())  # answered early: does not end the run
            if m == "hb":
                frames.append(_random_hb(rng, next_id))
            elif m == "keep":
                frames.append(keep_frame(_ids(rng, next_id, int(rng.integers(0, 11))), token=str(rng.choice(["u1", "u2", "s1", "bad"])),
                                         ms=int(rng.choice([0, 1000, 2000, 10000, 30000, 30001]))))
            elif m == "free":
                frames.append(free_frame(_ids(rng, next_id, int(rng.integers(0, 6))), token=str(rng.choice(["u1", "u1", "bad"]))))
            elif m == "wait":
                frames.append(wait_frame(token=str(rng.choice(["u1", "u2", "bad"])), env=int(rng.integers(0, 3)),
                                         imm=int(rng.integers(0, 5)), pre=int(rng.integers(0, 2)),
                                         ka_ms=int(rng.choice([1000, 3000, 10000, 30000])),
                                         ip=str(rng.choice(["172.16.0.1", "172.16.0.9", "10.7.0.3"]))))
            elif m == "config":
                frames.append(config_frame(str(rng.choice(["u1", "s1"]))))
            else:
                frames.append(running_frame())
    return frames


def run_random(t: Twins, seed: int, n_windows: int) -> int:
    """Seeded windows, ticks and roll-outs (the roll-out interval is 3 s).  Returns the number of frames."""
    rng = np.random.default_rng(seed)
    now, frames = 0.0, 0
    for _ in range(n_windows):
        now += float(rng.choice([0.0, 0.1, 0.5, 1.2, 3.1]))
        if rng.random() < 0.25:
            t.tick(now)
        w = random_window(rng, t.b.dispatcher.next_task_id())
        t.window(w, now)
        frames += len(w)
    return frames


# ---- targeted cases: each returns nothing and raises Mismatch (or AssertionError) if its rule is broken ---------------------
def _cluster(t: Twins, n=6, now=0.0, ms=5000):
    t.window([hb_frame(k, ms=ms) for k in range(n)], now)


def _grant(t: Twins, now: float, n=3, ka_ms=10000) -> list[int]:
    ans = t.window([wait_frame(imm=n, ka_ms=ka_ms, env=0)], now)
    body = PB["WaitForStartingTaskResponse"]()
    body.ParseFromString(ans[0][2])
    return [g.task_grant_id for g in body.grants]


def case_nat_cut(t: Twins):
    """Heartbeat 0 comes from 10.7.0.8 and reports 10.7.0.7:8335 (NAT); heartbeat 2 of the same run, itself behind NAT,
    registers 10.7.0.7:8335.  Heartbeat 0's notification must not find it (else the bookkeeper gains an entry under
    10.7.0.7:8335, which the exported state shows)."""
    _cluster(t, 4)
    ids = _grant(t, 0.5, 4)
    t.window([hb_frame(7, ip="10.7.0.8", running=ids[:2]), hb_frame(1, running=ids), hb_frame(9, ip="10.7.0.7", running=ids[2:]),
              hb_frame(8)], 1.0)
    t.window([running_frame()], 1.0)


def case_repeated_servant(t: Twins):
    """One servant twice in a run: the second notification sees the first's sweep."""
    _cluster(t, 3)
    ids = _grant(t, 0.5, 6)
    t.tick(11.0)  # the leases expire: zombies until a heartbeat leaves them out
    t.window([hb_frame(k, running=ids[:3]) for k in range(3)] + [hb_frame(k, running=ids[3:]) for k in range(3)], 11.5)
    t.window([running_frame(), keep_frame(ids)], 11.5)


def case_rejected_heartbeats(t: Twins):
    """Bad token, version below the minimum, unparsable location and a lease above 30 s inside one run."""
    _cluster(t, 2)
    t.window([hb_frame(3, token="bad"), hb_frame(4), hb_frame(5, version=1), hb_frame(6, location="not-an-endpoint"),
              hb_frame(7, ms=30001), hb_frame(8, ms=30000)], 1.0)
    assert t.a.dispatcher.num_servants() == 4


def case_last_length_wins(t: Twins, order=(20000, 2000)):
    """Two ids renewed by three frames of a run with different lengths: the last one sets the expiry.  At the boundary
    the first id is still alive (renewing it with length 0 succeeds); a nanosecond later the second is gone."""
    _cluster(t, 3, ms=30000)
    ids = _grant(t, 0.5, 2)
    now = 1.0
    t.window([keep_frame(ids, ms=order[0]), keep_frame(ids, ms=5000), keep_frame(ids, ms=order[1])], now)
    boundary = now + order[1] / 1000
    t.tick(boundary)
    ans = t.window([keep_frame(ids[:1], ms=0)], boundary)
    assert ans[0][2] == b"\x0a\x01\x01", ans
    t.tick(boundary + 1e-9)
    ans = t.window([keep_frame(ids[1:], ms=0)], boundary + 1e-9)
    assert ans[0][2] == b"\x0a\x01\x00", ans


def case_keepalive_edges(t: Twins):
    """Zombie, unknown, freed and never-issued ids in a keep-alive run, with lengths 0 and 30 s."""
    _cluster(t, 3)
    ids = _grant(t, 0.5, 4, ka_ms=1000)
    more = _grant(t, 0.5, 2, ka_ms=30000)
    t.tick(2.0)  # the first four are zombies now
    t.window([free_frame(more[:1])], 2.0)
    nxt = t.a.dispatcher.next_task_id()
    t.window([keep_frame(ids + [nxt, nxt + 1, 10**15], ms=0), keep_frame(more + [ids[0]], ms=30000),
              keep_frame(more[1:], ms=0, token="bad"), keep_frame(more, ms=30001), keep_frame([]),
              keep_frame(more[1:] * 3, ms=0)], 2.0)
    t.tick(2.0)
    t.tick(2.0 + 1e-9)


def case_free_run(t: Twins):
    """A FreeTask run with duplicated and unknown ids, then a solve that shows running_tasks."""
    _cluster(t, 2)
    ids = _grant(t, 0.5, 8)
    t.window([free_frame(ids[:3] + ids[:1]), free_frame([10**9, ids[1]]), free_frame(ids[3:4], token="bad"),
              free_frame(ids[4:5] * 2), unknown_frame(), free_frame([])], 1.0)
    t.window([wait_frame(imm=8, env=0)], 1.0)


def case_token_roll(t: Twins):
    """A roll-out that falls due at the run's `now`: every accepted heartbeat of the run gets the rolled window."""
    _cluster(t, 2)
    now = ROLLOUT_S + 0.5
    t.window([hb_frame(2, token="bad"), hb_frame(0), hb_frame(1), config_frame(), hb_frame(3)], now)
    t.window([config_frame()], now + ROLLOUT_S + 1.0)


TARGETED = {"nat_cut": case_nat_cut, "repeated_servant": case_repeated_servant,
            "rejected_heartbeats": case_rejected_heartbeats, "last_length_wins": case_last_length_wins,
            "last_length_wins_longer": lambda t: case_last_length_wins(t, order=(2000, 20000)),
            "keepalive_edges": case_keepalive_edges, "free_run": case_free_run, "token_roll": case_token_roll}


# ---- yd_keep_tasks_alive against the loop of yd_keep_task_alive -----------------------------------------------------------
def keep_tasks_alive_case(make, seed: int, make_a=None):
    """Twin dispatchers: one (`make_a`, by default `make`) takes yd_keep_tasks_alive, the other the same ids one
    yd_keep_task_alive call each.  The flags, and the leases' fate over the ticks that follow, must be the same."""
    rng = np.random.default_rng(seed)
    t = Twins(make_a or make, make)
    try:
        _cluster(t, 4)
        ids = _grant(t, 0.5, 6, ka_ms=1000) + _grant(t, 0.5, 6, ka_ms=30000)
        t.tick(2.0)  # the first six are zombies
        t.window([free_frame(ids[6:8])], 2.0)
        da, db = t.a.dispatcher, t.b.dispatcher
        nxt = db.next_task_id()
        pool = ids + [nxt, nxt + 3, 10**13]
        for step in range(4):
            now = 2.0 + step
            sel = [pool[int(i)] for i in rng.integers(0, len(pool), size=24)]
            lens = [float(rng.choice([0.0, 0.5, 1.0, 3.0, 30.0])) for _ in sel]
            got = da.keep_tasks_alive(sel, lens, now=now)
            want = np.array([db.keep_task_alive(i, x, now=now) for i, x in zip(sel, lens)])
            if not (got == want).all():
                raise Mismatch(f"keep_tasks_alive flags differ at step {step}")
            t.compare(now)
            for dt in (0.5, 1.0, 1.0 + 1e-9):
                t.tick(now + dt)
    finally:
        t.close()
