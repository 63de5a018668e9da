#!/usr/bin/env python
"""Host time of a window of Heartbeat, KeepTaskAlive or FreeTask frames served as one run by yd_wire_handle_frames,
against the same frames through yd_wire_call one by one.

Load: cfg2-mod's 2 000 servants holding the 100 k leases of one solve, on twin schedulers (one per path).  Windows:
2 000 Heartbeat frames x 50 running tasks, 10 000 KeepTaskAlive frames x 10 ids, 10 000 FreeTask frames x 10 ids.  The
two paths alternate in one process; every repetition's answers are compared frame by frame (status, description,
body).  Only the native calls are timed: the frames and arguments are built before the clock starts, and the
one-by-one loop includes a Python ctypes call per frame.  The FreeTask window releases its leases on the first (warm-up) repetition, so the timed ones free ids that are no
longer leased.  On a group (--world W, ranks as threads on ONE GPU over the test-only NCCL stand-in), every rank's
service is fed the window; the time is the slowest rank's.  One JSON line with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
FAKE = C.CDLL(str(ROOT / "tests" / "fake_nccl" / "libnccl.so.2"), mode=C.RTLD_GLOBAL)  # before anything loads NCCL

import numpy as np  # noqa: E402

sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import service_runs_cases as R  # noqa: E402
from yadcc_b200 import _abi  # noqa: E402
from yadcc_b200 import streams as S  # noqa: E402
from yadcc_b200._abi import GRANT_DTYPE  # noqa: E402
from yadcc_b200.dispatcher import TaskDispatcher  # noqa: E402
from yadcc_b200.service import SchedulerService  # noqa: E402


def par(fns):
    out = [None] * len(fns)
    ts = [threading.Thread(target=lambda i=i, f=f: out.__setitem__(i, f())) for i, f in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


class _GroupView:
    native = True

    def __init__(self, local):
        self.local = local


def loaded(lib, w, world):
    """`world` rank handles (a plain handle for world 0) with cfg2-mod registered and its 100 k leases granted, and
    their services.  Returns (ranks, services, granted ids, their servants)."""
    n = max(world, 1)
    ranks = [TaskDispatcher(lib) for _ in range(n)]
    if world:
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        assert lib.yd_shard_unique_id(uid) == 0
        assert par([lambda r=r: lib.yd_shard_init(ranks[r]._h, r, n, uid) for r in range(n)]) == [0] * n
    for d in ranks:
        w.register(d, now=0.0, expires_in=30.0)
    full = w.build_requests(ranks[0])
    cuts = [len(full) * g // n for g in range(n + 1)]
    parts = [np.ascontiguousarray(full[cuts[r]:cuts[r + 1]]) for r in range(n)]
    outs = [np.zeros(max(len(p), 1), dtype=GRANT_DTYPE) for p in parts]
    if world:
        assert par([lambda r=r: lib.yd_shard_wait_for_starting_new_tasks(ranks[r]._h, 1_000_000, parts[r].ctypes.data,
                                                                          len(parts[r]), outs[r].ctypes.data)
                    for r in range(n)]) == [0] * n
    else:
        outs[0] = ranks[0].wait_for_starting_new_tasks(full, now=0.001)
    g = np.concatenate([outs[r][:len(parts[r])] for r in range(n)])
    ok = g["status"] == _abi.STATUS_GRANTED
    kw = dict(acceptable_user_tokens="u1", acceptable_servant_tokens="s1", token_seed=3, now=0.0)
    svcs = par([lambda d=d: SchedulerService(_GroupView(d) if world else d, **kw) for d in ranks])
    return ranks, svcs, g["task_id"][ok], g["servant_index"][ok]


class RunCall:
    """One yd_wire_handle_frames over a window, its inputs built before the clock starts."""

    def __init__(self, svc, wire):
        self.lib, self.h, self.n = svc._lib, svc._h, len(wire)
        self.keep = [(C.create_string_buffer(f, len(f)), ip.encode()) for f, ip in wire]
        self.ins = (_abi.yd_wire_in * self.n)()
        for i, (buf, ip) in enumerate(self.keep):
            self.ins[i] = _abi.yd_wire_in(C.cast(buf, C.c_void_p), len(wire[i][0]), ip, 0, 0)
        self.cap = 512 * self.n + (1 << 20)
        self.out = C.create_string_buffer(self.cap)
        self.outs = (_abi.yd_wire_out * self.n)()

    def time(self, now_ns):
        t0 = time.perf_counter()
        total = self.lib.yd_wire_handle_frames(self.h, now_ns, self.ins, self.n, C.cast(self.out, C.c_void_p), self.cap,
                                               self.outs)
        dt = (time.perf_counter() - t0) * 1e3
        assert total != (1 << 64) - 1
        return dt

    def answers(self):
        raw = self.out.raw
        return [raw[o.offset:o.offset + o.len] for o in self.outs]


class OneByOne:
    """The same frames' bodies through yd_wire_call, one call each, the arguments built before the clock starts."""

    def __init__(self, svc, frames):
        self.lib, self.h = svc._lib, svc._h
        self.args = [((R.W.SERVICE + f.method).encode(), f.ip.encode(), f.body) for f in frames]
        self.cap = 1 << 20
        self.out = C.create_string_buffer(self.cap)
        self.answers = []

    def time(self, now_ns):
        n, desc = C.c_size_t(0), C.c_char_p()
        got = []
        t0 = time.perf_counter()
        for m, ip, body in self.args:
            st = self.lib.yd_wire_call(self.h, now_ns, m, ip, 0, body, len(body), C.cast(self.out, C.c_void_p), self.cap,
                                       C.byref(n), C.byref(desc))
            got.append((st, desc.value, C.string_at(self.out, n.value)))
        dt = (time.perf_counter() - t0) * 1e3
        self.answers = [(st, (d or b"").decode(), b) for st, d, b in got]
        return dt


def windows(w, d, ids, srv):
    by = {}
    for t, s in zip(ids.tolist(), srv.tolist()):
        by.setdefault(s, []).append(t)
    hb = []
    for i, sv in enumerate(w.servants):
        loc = d.servant_location(i)
        m = R.PB["HeartbeatRequest"](token="s1", next_heartbeat_in_ms=30000, version=sv.version, location=loc,
                                     num_processors=sv.num_processors, capacity=sv.max_tasks, servant_priority=2,
                                     total_memory_in_bytes=sv.total_memory_in_bytes,
                                     memory_available_in_bytes=sv.memory_available_in_bytes)
        for e in sv.environments:
            m.env_descs.add().compiler_digest = e
        for j, t in enumerate(by.get(i, [])[:50]):
            r = m.running_tasks.add()
            r.servant_task_id, r.task_grant_id, r.servant_location, r.task_digest = j + 1, t, loc, f"{t:064x}"
        hb.append(R.Frame("Heartbeat", m.SerializeToString(), loc.rsplit(":", 1)[0]))
    ka = [R.keep_frame(ids[k * 10:(k + 1) * 10], ms=20000) for k in range(10_000)]
    fr = [R.free_frame(ids[k * 10:(k + 1) * 10]) for k in range(10_000)]
    return {"heartbeat": hb, "keep_task_alive": ka, "free_task": fr}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--worlds", default="0,1,2,4", help="0: one handle; W > 0: a group of W ranks")
    ap.add_argument("--library", default=None, help="another library for one handle (a rehearsal on a CPU checker)")
    a = ap.parse_args()
    lib = a.library or _abi.load_library()
    w = S.config2(variant="mod")
    smi = [] if a.library else subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": smi[0] if smi else None, "reps": a.reps, "load": "cfg2-mod: 2000 servants, 100 k leases", "results": {}}
    for world in [int(x) for x in a.worlds.split(",")]:
        A, B = loaded(lib, w, world), loaded(lib, w, world)
        assert (A[2] == B[2]).all()
        wins = windows(w, A[0][0], A[2], A[3])
        res = {}
        for name, frames in wins.items():
            wire = [(R._frame(f, k + 1), f.ip) for k, f in enumerate(frames)]
            runs = [RunCall(s, wire) for s in A[1]]
            ones = [OneByOne(s, frames) for s in B[1]]
            t_run, t_one = [], []
            for rep in range(a.reps + 1):
                now_ns = 1_000_000_000 + rep * 10_000_000
                t_run.append(max(par([lambda c=c: c.time(now_ns) for c in runs])))
                t_one.append(max(par([lambda c=c: c.time(now_ns) for c in ones])))
                outs, ans = [c.answers() for c in runs], [c.answers for c in ones]
                for r in range(len(runs)):
                    assert outs[r] == outs[0] and ans[r] == ans[0], (name, rep, r)
                for k, (o, (st, desc, body)) in enumerate(zip(outs[0], ans[0])):
                    assert R._parse(o) == (st, desc if st else "", body if st == 0 else b""), (name, rep, k)
                print(f"{name} W={world} rep {rep}: {t_run[-1]:.2f} ms as a run, {t_one[-1]:.2f} ms one by one", file=sys.stderr,
                      flush=True)
            t_run, t_one = t_run[1:], t_one[1:]  # the first repetition warms up
            res[name] = {"frames": len(frames),
                         "run_ms": round(float(np.median(t_run)), 2), "run_range_ms": [round(min(t_run), 2), round(max(t_run), 2)],
                         "one_by_one_ms": round(float(np.median(t_one)), 2),
                         "one_by_one_range_ms": [round(min(t_one), 2), round(max(t_one), 2)]}
        out["results"]["handle" if world == 0 else f"group W={world}"] = res
        for ranks, svcs, _, _ in (A, B):
            for s in svcs:
                s.close()
            for d in ranks:
                if world:
                    lib.yd_shard_finalize(d._h)
                d.close()
    out["note"] = "groups are threads on one GPU over the test-only NCCL stand-in; real NCCL over several GPUs is not measured"
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
