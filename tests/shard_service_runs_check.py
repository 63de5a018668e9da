#!/usr/bin/env python
"""Runs of Heartbeat, KeepTaskAlive and FreeTask frames on a range-sharded group's services (yd_shard_service_create),
W ranks as W threads of one process over the test-only NCCL stand-in (tests/fake_nccl/libnccl.so.2, loaded with
RTLD_GLOBAL before anything else; this process must not import torch).

  * streams: the seeded windows of tests/service_runs_cases.py go to every rank's service through
    yd_wire_handle_frames, and frame by frame through yd_wire_call to one service over the CPU checker
    (checkers/libydport_state.so).  Every rank's response bytes must be the same, and each frame's status,
    description and body must equal the checker's; after every window the servant state, next task id and lease
    count must match (the group's leases summed over the ranks).
  * collectives: a run of 1, 8 or 64 frames of one method costs every rank the same number of collectives, counted
    by the stand-in's yd_fake_nccl_stats.
  * yd_shard_keep_tasks_alive against the checker's yd_keep_tasks_alive: flags and the leases' fate over ticks.

Prints one JSON line per case and a final {"shard_service_runs": ...} line; exit code 0 iff everything matched.
"""
import argparse
import ctypes as C
import json
import sys
import threading
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE = C.CDLL(str(ROOT / "tests" / "fake_nccl" / "libnccl.so.2"), mode=C.RTLD_GLOBAL)
CHECKER = ROOT / "checkers" / "libydport_state.so"

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import service_runs_cases as R  # noqa: E402
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200.dispatcher import TaskDispatcher  # noqa: E402
from yadcc_b200.service import SchedulerService  # noqa: E402

assert "torch" not in sys.modules, "torch loads the real libnccl.so.2"


def par(fns):
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


class _GroupView:
    """What SchedulerService needs of a RangeShardedDispatcher, without torch: the rank handle, joined to the group."""

    native = True

    def __init__(self, local):
        self.local = local


def collectives(r: int) -> int:
    a = (C.c_ulonglong * 4)()
    FAKE.yd_fake_nccl_stats(r, a)
    return int(a[0])


class Group:
    def __init__(self, world: int, seed: int = 5):
        self.W = world
        self.lib = _abi.load_library()
        self.ranks = [TaskDispatcher(self.lib) for _ in range(world)]
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        assert self.lib.yd_shard_unique_id(uid) == 0
        assert par([lambda r=r: self.lib.yd_shard_init(self.ranks[r]._h, r, world, uid) for r in range(world)]) == [0] * world
        self.checker = TaskDispatcher(str(CHECKER))
        kw = dict(acceptable_user_tokens=R.USER, acceptable_servant_tokens=R.SERVANT, min_daemon_version=R.MIN_VERSION,
                  serving_daemon_token_rollout_interval=R.ROLLOUT_S, token_seed=seed, now=0.0)
        self.svcs = par([lambda d=d: SchedulerService(_GroupView(d), **kw) for d in self.ranks])
        self.one = SchedulerService(self.checker, **kw)
        self.corr = 0
        self.windows = 0

    def close(self):
        for s in self.svcs:
            s.close()
        self.one.close()
        for d in self.ranks:
            self.lib.yd_shard_finalize(d._h)
            d.close()
        self.checker.close()

    def window(self, frames, now):
        wire = []
        for f in frames:
            self.corr += 1
            wire.append((R._frame(f, self.corr), f.ip))
        outs = par([lambda s=s: s.handle_frames(wire, now=now) for s in self.svcs])
        for r in range(1, self.W):
            if outs[r] != outs[0]:
                raise R.Mismatch(f"window {self.windows}: rank {r}'s bytes differ from rank 0's")
        answers = []
        for k, (f, o) in enumerate(zip(frames, outs[0])):
            st, desc, body = self.one.call(R.W.SERVICE + f.method, f.body, f.ip, now=now)
            want = (st, desc if st else "", body if st == 0 else b"")
            if o[0] != 1 or R._parse(o[3]) != want:
                raise R.Mismatch(f"window {self.windows} frame {k} ({f.method}): group {R._parse(o[3])!r} != one {want!r}")
            answers.append(want)
        self.compare()
        self.windows += 1
        return answers

    def tick(self, now):
        for d in self.ranks + [self.checker]:
            d.on_expiration_timer(now=now)
        self.compare()

    def compare(self):
        ref = self.checker.servant_state()
        for r, d in enumerate(self.ranks):
            st = d.servant_state()
            if len(st) != len(ref):
                raise R.Mismatch(f"after window {self.windows}: rank {r}'s servant count differs")
            for f in ("running_tasks", "ever_assigned_tasks", "capacity_available", "expires_at_ns"):
                if (st[f] != ref[f]).any():
                    raise R.Mismatch(f"after window {self.windows}: rank {r}'s {f} differs")
            if d.next_task_id() != self.checker.next_task_id():
                raise R.Mismatch(f"after window {self.windows}: rank {r}'s next task id differs")
        if sum(d.num_tasks() for d in self.ranks) != self.checker.num_tasks():
            raise R.Mismatch(f"after window {self.windows}: the group's lease count differs")


def run_streams(world, seeds, n_windows):
    out = {"case": "streams", "world": world, "ok": True, "frames": 0}
    for seed in seeds:
        g = Group(world, seed)
        try:
            rng = np.random.default_rng(seed)
            now = 0.0
            for _ in range(n_windows):
                now += float(rng.choice([0.0, 0.1, 0.5, 1.2, 3.1]))
                if rng.random() < 0.25:
                    g.tick(now)
                w = R.random_window(rng, g.checker.next_task_id())
                g.window(w, now)
                out["frames"] += len(w)
        except R.Mismatch as e:
            out.update(ok=False, seed=seed, error=str(e))
        finally:
            g.close()
        if not out["ok"]:
            break
    print(json.dumps(out), flush=True)
    return out["ok"]


def run_collectives(world):
    """One window per (method, run length); the collectives each costs on every rank must not depend on the length."""
    out = {"case": "collectives", "world": world, "ok": True, "per_run": {}}
    g = Group(world)
    try:
        g.window([R.hb_frame(k, ms=30000) for k in range(6)], 0.0)
        ids = [x for _ in range(6) for x in _granted(g.window([R.wait_frame(imm=4)], 0.1))]
        for method in ("Heartbeat", "KeepTaskAlive", "FreeTask"):
            counts = {}
            for n in (1, 8, 64):
                if method == "Heartbeat":
                    frames = [R.hb_frame(k % 6, ms=30000, running=ids[k % 6::6]) for k in range(n)]
                elif method == "KeepTaskAlive":
                    frames = [R.keep_frame(ids[k % len(ids):][:5] + [10**9], ms=1000 + 100 * (k % 3)) for k in range(n)]
                else:
                    frames = [R.free_frame([10**9 + k, 10**10]) for k in range(n)]
                before = [collectives(r) for r in range(world)]
                g.window(frames, 0.2)
                after = [collectives(r) for r in range(world)]
                d = [a - b for a, b in zip(after, before)]
                if len(set(d)) != 1:
                    raise R.Mismatch(f"{method} x {n}: ranks made different numbers of collectives {d}")
                counts[n] = d[0]
            out["per_run"][method] = counts
            if len(set(counts.values())) != 1 or counts[1] < 1:
                raise R.Mismatch(f"{method}: collectives per run depend on its length: {counts}")
    except R.Mismatch as e:
        out.update(ok=False, error=str(e))
    finally:
        g.close()
    print(json.dumps(out), flush=True)
    return out["ok"]


def _granted(answers):
    body = R.PB["WaitForStartingTaskResponse"]()
    body.ParseFromString(answers[0][2])
    return [x.task_grant_id for x in body.grants]


def run_keep_tasks_alive(world, seed):
    out = {"case": "keep_tasks_alive", "world": world, "ok": True, "calls": 0}
    rng = np.random.default_rng(seed)
    g = Group(world, seed)
    try:
        g.window([R.hb_frame(k, ms=30000) for k in range(6)], 0.0)
        ids = _granted(g.window([R.wait_frame(imm=12, ka_ms=1000)], 0.5)) + _granted(
            g.window([R.wait_frame(imm=12, ka_ms=30000)], 0.5))
        g.tick(2.0)  # the first dozen are zombies
        g.window([R.free_frame(ids[12:14])], 2.0)
        nxt = g.checker.next_task_id()
        pool = ids + [nxt, nxt + 2, 10**13]
        lib = g.lib
        for step in range(5):
            now = 2.0 + step
            sel = [pool[int(i)] for i in rng.integers(0, len(pool), size=500)]
            lens = [float(rng.choice([0.0, 0.5, 1.0, 3.0, 30.0])) for _ in sel]
            got = par([lambda d=d: d._keep_alive_with(lib.yd_shard_keep_task_alive, sel, lens, now,
                                                       fn_each=lib.yd_shard_keep_tasks_alive) for d in g.ranks])
            want = g.checker.keep_tasks_alive(sel, lens, now=now)
            for r in range(world):
                if not (got[r] == want).all():
                    raise R.Mismatch(f"step {step}: rank {r}'s flags differ")
            out["calls"] += 1
            g.compare()
            for dt in (0.5, 1.0, 1.0 + 1e-9):
                g.tick(now + dt)
    except R.Mismatch as e:
        out.update(ok=False, error=str(e))
    finally:
        g.close()
    print(json.dumps(out), flush=True)
    return out["ok"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--seeds", default="1,2,3")
    ap.add_argument("--windows", type=int, default=30)
    a = ap.parse_args()
    ok = run_streams(a.world, [int(x) for x in a.seeds.split(",") if x], a.windows)
    ok = run_collectives(a.world) and ok
    ok = run_keep_tasks_alive(a.world, 40 + a.world) and ok
    print(json.dumps({"shard_service_runs": ok, "world": a.world, "torch_loaded": "torch" in sys.modules}), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
