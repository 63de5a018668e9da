"""Cases at both sides of every rule by which the merge solver hands a component back to the sequential solver
(yadcc_b200/csrc/solve_merge.cuh), shared by the CPU model test (test_merge_walk_model.py), the GPU test
(test_merge_handback.py) and, for the range-sharded record window (SHARDED), shard_merge_check.py.

Every case is one batch on a fresh cluster of one coupled component.  `back` is the reason mask the solve's
YDSCHED_DEBUG line reports as merge_back (solve_merge.cuh kBack*), `edge` what the plain model of the walk
(merge_walk_model.py) must show for the case to sit where its name says, and `chunk` the YDSCHED_MERGE_CHUNK the GPU
side runs it with.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

import numpy as np

from yadcc_b200 import PRIORITY_DEDICATED, PRIORITY_USER, STATUS_TIMEOUT, Servant
from yadcc_b200 import streams as S

GiB = 1 << 30
MERGE_PEND = 8          # kMergePend
MERGE_SKIP = 1 << 20    # kMergeSkipMax
BACK_PEND, BACK_SKIP, BACK_CHECK = 1, 2, 8  # kBackPend, kBackSkip, kBackCheck
D, D2 = "6d" * 32, "7e" * 32
BIG_CHUNK = 1 << 21     # one chunk per component: the long pending run is served in one warp's walk


@dataclass
class Case:
    servants: list
    reqs: list                        # (digest, min_version, requestor IP) in FIFO order
    back: int                         # merge_back of the solve
    edge: Callable                    # Walk -> bool
    chunk: int = 0                    # YDSCHED_MERGE_CHUNK (0: the default)
    merge: bool = True                # the merge solver runs (False: the component is the sequential solver's)


def _sv(i, nproc, *, envs=(D,), version=8, dedicated=False, max_tasks=None, memory=(0, 0)):
    return Servant(f"{S.servant_ip(i)}:8335", None, list(envs), version, nproc, 0, memory[0], memory[1],
                   nproc if max_tasks is None else max_tasks, PRIORITY_DEDICATED if dedicated else PRIORITY_USER)


def _x(i):
    return f"172.30.{(i >> 8) & 255}.{i & 255}"  # a requestor that is no servant


A = S.servant_ip(0)  # the own IP of servant 0 in every case


def pend_case(runs: int, k: int, lead: int = 0) -> Case:
    """Servant 0 is the only dedicated one: its tier-0 slots lead the sorted order.  After `lead` requests from other
    IPs the queue alternates its IP with another one, `runs` pairs, the pairs' classes (min_version 8, 7, ...) taking
    turns over `k` classes: every tier-0 slot of servant 0 passes over one request of its own and leaves one run.  Four
    user servants of 64 slots serve the runs afterwards.  With `lead` = 24 and chunks of 32 slots, runs 1-8 are made in
    the first chunk and the second starts from a carried state that holds them."""
    tier0 = lead + runs + 4
    svs = [_sv(0, 2 * tier0, dedicated=True)] + [_sv(i, 64) for i in range(1, 5)]
    mv = lambda i: 8 - i % k  # noqa: E731
    reqs = [(D, mv(i), _x(i)) for i in range(lead)]
    for i in range(runs):
        reqs += [(D, mv(i), A), (D, mv(i), _x(lead + i))]
    reqs += [(D, mv(i), _x(100 + i)) for i in range(40)]
    return Case(svs, reqs, BACK_PEND if runs > MERGE_PEND else 0, lambda w: w.pend == runs and not w.blocking,
                chunk=32 if lead else 0)


def contiguous_case(n: int) -> Case:
    """The first slot passes over `n` consecutive requests of its own servant: one run however long."""
    svs = [_sv(0, 8, dedicated=True)] + [_sv(i, 64) for i in range(1, 5)]
    reqs = [(D, 8, A)] * n + [(D, 8, _x(i)) for i in range(60)]
    return Case(svs, reqs, 0, lambda w: w.pend == 1 and w.skip == n and not w.blocking)


def skip_case(length: int, at_end: bool) -> Case:
    """Servant 0 holds one tier-0 slot, the first of the walk; `length` requests from its IP head the queue, then (not
    `at_end`) one from another IP.  Four user servants hold enough slots for every request, so nothing is left over."""
    svs = [_sv(0, 1, dedicated=True)] + [_sv(i, (1 << 18) + 1) for i in range(1, 5)]
    reqs = [(D, 8, A)] * length + ([] if at_end else [(D, 8, _x(0))])
    return Case(svs, reqs, BACK_SKIP if length > MERGE_SKIP else 0, lambda w: w.skip == length and not w.blocking,
                chunk=BIG_CHUNK)


def check_case(kind: str) -> Case:
    """A saturated class: servant 0 (own IP A, 3 slots) and servant 1 (1 slot).  The request from A is left unserved;
    the last-resort rule (cc:394-396) hands the component back when a slot of servant 0 went to a later request or
    stayed free, and must ignore an own servant that could not serve the request anyway."""
    x = lambda i, mv=8, d=D: (d, mv, _x(i))  # noqa: E731
    a = (D, 8, A)
    blocking = lambda w: len(w.blocking) == 1  # noqa: E731
    if kind == "earlier":   # every slot of servant 0 went to an earlier request
        return Case([_sv(0, 3), _sv(1, 1)], [x(0), x(1), x(2), x(3), a], 0, lambda w: not w.blocking and w.status[4] == STATUS_TIMEOUT)
    if kind == "later":     # its last slot went to a later request
        return Case([_sv(0, 3), _sv(1, 1)], [x(0), x(1), a, x(3), x(4)], BACK_CHECK, blocking)
    if kind == "free":      # its last slot stayed free
        return Case([_sv(0, 3), _sv(1, 1)], [x(0), x(1), a, x(3)], BACK_CHECK, blocking)
    # servant 0 is free but cannot take the request: a slot of it stays free and the request stays unserved
    if kind == "version":   # version below the class's min_version (it serves the min_version-7 class)
        svs = [_sv(0, 2, version=7), _sv(1, 1)]
        reqs = [x(0), a, x(2, mv=7)]
    elif kind == "digest":  # without the digest (it serves the other one)
        svs = [_sv(0, 2, envs=(D2,)), _sv(1, 1, envs=(D, D2))]
        reqs = [x(0), a, x(2, d=D2)]
    elif kind == "max-tasks":
        svs = [_sv(0, 2, max_tasks=0), _sv(1, 1)]
        reqs = [x(0), a]
    elif kind == "low-memory":
        svs = [_sv(0, 2, memory=(64 * GiB, GiB)), _sv(1, 1)]
        reqs = [x(0), a]
    else:
        raise ValueError(kind)
    return Case(svs, reqs, 0, lambda w: not w.blocking and w.status[1] == STATUS_TIMEOUT)


def classes_case(k: int) -> Case:
    """`k` classes (min_version 1 .. k) on one component with requests from a servant's own IP: the merge solver takes
    up to 32 of them (classes.cuh), the sequential solver more."""
    rng = np.random.default_rng(k)
    svs = [_sv(i, 64, version=40) for i in range(4)]
    reqs = [(D, 1 + i % k, S.servant_ip(int(rng.integers(0, 4))) if rng.random() < 0.2 else _x(i)) for i in range(300)]
    return Case(svs, reqs, 0, lambda w: len(w.list_len) == k and not w.blocking, merge=k <= 32)


RQ_MARGIN = 1024  # kRqMargin: a range-sharded rank gathers a class's records [0, slot-list length + margin)


def margin_case(past: int) -> Case:
    """Range-sharded window: the walk reads class c1's record `past` places behind its slot list (len + 1023: every
    record it reads was gathered; len + 1024: it was not, and every rank falls back to the whole queue).

    Servant 0 (own IP A) serves c1 (min_version 8) and c2 (min_version 9), servants 1-4 (version 8) c1 only.  Servant 0's
    first slot takes the first request; the others' slots below half their capacity take the next 2c; then servant 0's
    second slot meets a head of c1 from its own IP with nothing but its own requests behind it: the one-slot step walks to
    the end of c1's list and the slot takes the one c2 request, which sits between the requests of A that the
    remaining slots serve and those left over (so no blocking pair forms)."""
    c = 512
    svs = [_sv(0, 2, version=9)] + [_sv(i, c) for i in range(1, 5)]
    n1 = (4 * c + 2) + past + 1  # c1's requests: its slot-list length + past + 1
    reqs = [(D, 8, _x(i)) for i in range(1 + 2 * c)] + [(D, 8, A)] * (n1 - 1 - 2 * c)
    reqs.insert(3 * c, (D, 9, _x(9999)))
    return Case(svs, reqs, 0, lambda w: w.margin() == past and not w.blocking)


def saturated_case() -> Case:
    """A saturated class on a large component: c1 (min_version 9) is served by servant 0 alone (64 slots) and asked for
    3000 times, c2 (min_version 8) by 16 servants of 512 slots.  The walk reads c1's records only up to its slot list,
    far inside a range-sharded rank's window; chunks far down the slot list start from a guessed state whose c1 head lies
    beyond that window."""
    rng = np.random.default_rng(3)
    svs = [_sv(0, 64, version=9)] + [_sv(i, 512) for i in range(1, 17)]
    reqs = [(D, 9 if rng.random() < 0.5 else 8, _x(i)) for i in range(6000)]
    return Case(svs, reqs, 0, lambda w: w.margin() < 0 and not w.blocking)


SHARDED = {"margin-1023": margin_case(RQ_MARGIN - 1), "margin-1024": margin_case(RQ_MARGIN), "saturated": saturated_case()}

CASES = {
    **{f"pend-{n}-k{k}": pend_case(n, k) for n in (8, 9) for k in (1, 2, 3)},
    **{f"pend-{n}-k{k}-chunk32": pend_case(n, k, lead=24) for n in (8, 9) for k in (1, 2, 3)},
    "contiguous-9": contiguous_case(9),
    **{f"skip-{where}-{n}": skip_case(n, where == "end") for where in ("head", "end") for n in (MERGE_SKIP, MERGE_SKIP + 1)},
    **{f"check-{k}": check_case(k) for k in ("earlier", "later", "free", "version", "digest", "max-tasks", "low-memory")},
    "classes-32": classes_case(32),
    "classes-33": classes_case(33),
}
ALL = {**CASES, **SHARDED}


def stream(d, case: Case) -> S.Stream:
    """Heartbeats, the batch, the servants' state."""
    envs = {e: d.intern_env(e) for e in (D, D2)}
    ips = {ip: d.intern_ip(ip) for ip in sorted({ip for _, _, ip in case.reqs})}
    env = np.fromiter((envs[e] for e, _, _ in case.reqs), np.uint32, len(case.reqs))
    ip = np.fromiter((ips[x] for _, _, x in case.reqs), np.uint32, len(case.reqs))
    mv = np.fromiter((m for _, m, _ in case.reqs), np.uint32, len(case.reqs))
    ev = [("hb", 0.0, sv, 100.0) for sv in case.servants]
    ev += [("wait", 0.001, S._requests(d, env, ip, mv)), ("state",)]
    return S.Stream("merge-handback", ev)
