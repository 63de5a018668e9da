"""A plain model of the merge solver's slot-side walk (yadcc_b200/csrc/solve_merge.cuh, header), without its limits.

One batch on a fresh cluster (running_tasks = 0), one coupled component.  The slots of every servant are walked in the
common sorted order (tier, r / cap(r), registry position) -- the slot-key model of key_cases.py -- and each slot takes
the earliest unserved request of the classes its servant is eligible for whose own servant is not this one.  Requests
a slot passes over stay pending as [j0, j1) runs of a class's FIFO list per (class, servant); a pending run is served
before the class's head; a pass contiguous with the class's latest run of the same servant extends it.

Besides the decisions the walk reports the high-water marks each hand-back rule of the kernel tests:
  pend    pending runs held at once (kMergePend)
  skip    the longest run of own-servant records walked over, counted after each step as the one-slot step counts it,
          so a run that reaches the end of a class's list counts too (kMergeSkipMax)
  read    per class, the highest record index read: with the class's slot-list length, the range-sharded window
          (kRqMargin)
  merges  passes that extended a run instead of opening one
and the requests that form a blocking pair with their own servant (the last-resort rule, k_merge_check).
"""
from __future__ import annotations

from dataclasses import dataclass, field

from key_cases import _cap, _tier
from yadcc_b200 import STATUS_GRANTED, STATUS_TIMEOUT
from yadcc_b200._abi import STATUS_ENVIRONMENT_NOT_FOUND

MIN_MEMORY = 10 << 30  # servant_min_memory_for_accepting_new_task's default


@dataclass
class Walk:
    status: list[int]
    pick: list[int]                  # servant index, or -1
    pend: int = 0
    skip: int = 0
    merges: int = 0
    read: dict = field(default_factory=dict)      # class -> highest record index read
    list_len: dict = field(default_factory=dict)  # class -> slots of its eligible servants
    blocking: list[int] = field(default_factory=list)

    def margin(self) -> int:
        """How far past its slot list a class's records were read (the range-sharded window is len + kRqMargin)."""
        return max((self.read[c] - self.list_len[c] for c in self.read), default=-1)


def low_memory(sv) -> bool:
    return sv.total_memory_in_bytes != 0 and sv.memory_available_in_bytes < MIN_MEMORY


def slots(servants) -> list[tuple[int, int]]:
    """(servant, running_tasks) of every free slot of a fresh cluster, in the common sorted order."""
    out = []
    for i, sv in enumerate(servants):
        if low_memory(sv):
            continue  # capacity = running_tasks: never free
        r = 0
        while r < _cap(sv, r):
            out.append(((_tier(sv, r), r / _cap(sv, r), i), i, r))  # (the reference's double, as key_cases)
            r += 1
    return [(i, r) for _, i, r in sorted(out)]


def eligible(sv, digest: str, mv: int) -> bool:
    return digest in sv.environments and sv.max_tasks != 0 and sv.version >= mv


def walk(servants, reqs) -> Walk:
    """`reqs`: (digest, min_version, requestor IP) per request, in FIFO order."""
    ip_of = [sv.observed_location.split(":")[0] for sv in servants]
    own = [ip_of.index(ip) if ip in ip_of else -1 for _, _, ip in reqs]
    assert all(ip_of.count(ip) <= 1 for _, _, ip in reqs), "one servant per requestor IP (the merge solver's components)"
    classes = sorted({(d, mv) for d, mv, _ in reqs})
    queue = {c: [q for q, (d, mv, _) in enumerate(reqs) if (d, mv) == c] for c in classes}
    elig = {c: [eligible(sv, *c) for sv in servants] for c in classes}
    order = slots(servants)
    w = Walk([STATUS_TIMEOUT] * len(reqs), [-1] * len(reqs))
    w.list_len = {c: sum(elig[c][s] for s, _ in order) for c in classes}
    h = {c: 0 for c in classes}
    runs: list[list] = []  # [class, servant, j0, j1], per class in queue order
    taker: dict[int, list] = {}

    def read(c, j):
        w.read[c] = max(w.read.get(c, -1), j)

    for s, _ in order:
        if not any(elig[c][s] for c in classes):
            continue  # (in no class's slot list)
        best = None  # (request, class, pending run or None, end of the pass)
        for c in classes:
            if not elig[c][s]:
                continue
            q = c_run = None
            for run in runs:
                if run[0] == c and run[1] != s:
                    c_run = run
                    read(c, run[2])
                    q = queue[c][run[2]]
                    break
            j = h[c]
            if c_run is None:
                while j < len(queue[c]):
                    read(c, j)
                    if own[queue[c][j]] != s:
                        q = queue[c][j]
                        break
                    j += 1
                    w.skip = max(w.skip, j - h[c])
            if q is not None and (best is None or q < best[0]):
                best = (q, c, c_run, j)
        taker.setdefault(s, []).append(best[0] if best else None)
        if best is None:
            continue
        q, c, c_run, j = best
        w.status[q], w.pick[q] = STATUS_GRANTED, s
        if c_run is not None:
            c_run[2] += 1
            if c_run[2] == c_run[3]:
                runs.remove(c_run)
            continue
        if j > h[c]:
            last = [run for run in runs if run[0] == c]
            if last and last[-1][1] == s and last[-1][3] == h[c]:
                last[-1][3] = j
                w.merges += 1
            else:
                runs.append([c, s, h[c], j])
                w.pend = max(w.pend, len(runs))
        h[c] = j + 1
    for q, (d, mv, _) in enumerate(reqs):
        if not any(elig[(d, mv)]):
            w.status[q] = STATUS_ENVIRONMENT_NOT_FOUND
            continue
        o = own[q]
        if w.status[q] != STATUS_TIMEOUT or o < 0 or o not in taker or not eligible(servants[o], d, mv):
            continue
        # a slot of the own servant went to a later request, or stayed free: it would have taken this one
        if max(len(reqs) if t is None else t for t in taker[o]) > q:
            w.blocking.append(q)
    return w
