"""Slot-key precision at the narrow / wide key limit (common.cuh kNarrowCapLimit = 8192).

A servant's pick key at running_tasks r is (tier, r / cap(r), registry position) (task_dispatcher.cc:405-451).  The
CUDA backend orders it by floor(r * 2^27 / cap) while every capacity is <= 8192 and by the reference's own double
r / cap above that.  Two 27-bit floors of distinct fractions can only coincide when cap1 * cap2 > 2^27, i.e. for
capacities above ~11 585, so the limit is conservative; the clusters below sit on both sides of it and at 16 k, where a
narrow key would merge (and so misorder) neighbouring slots.

Each cluster has ten servants of one digest: capacities near the limit, loads (cap changes with r for r < load),
dedicated servants with odd nproc (the tier boundary 2r < nproc falls between two slots) and two servants whose
capacities repeat earlier ones (equal fractions: registry position breaks the tie).  `model_walk` replays
UnsafePickServantFor with Python floats -- the reference's IEEE doubles -- and `check_walk` uses exact fractions to
show that a walk without self-IP requests visits the slots in increasing (tier, r / cap, position) order and reaches
the edge its cluster is meant to test.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from yadcc_b200 import PRIORITY_DEDICATED, PRIORITY_USER, STATUS_GRANTED, STATUS_TIMEOUT, Servant
from yadcc_b200 import streams as S

DIGEST = "4b" * 32
N_WALK = 70_000   # requests of the long batch: it walks 70 k of the cluster's 82 k / 164 k slots
N_SELF = 10_000   # a second batch, 10 % of it from servants' own IPs (their own slot is the last resort)
CLUSTERS = {"narrow-8192": (8185, 8192), "wide-8193": (8186, 8193), "wide-16384": (16377, 16384)}


def key_servants(lo: int, hi: int) -> list[Servant]:
    caps = list(range(lo, hi + 1)) + [hi, lo]  # the last two repeat the capacities of servants 7 and 0
    out = []
    for k, c in enumerate(caps):
        dedicated = k in (1, 4, 6)
        nproc = c - (1 - c % 2) if dedicated else c  # odd: 2r < nproc flips between r = (nproc-1)/2 and (nproc+1)/2
        load = {2: 1500, 3: 300, 5: 4000}.get(k, 0)  # cap(r) = nproc - load + r below r = load
        out.append(Servant(f"10.77.0.{k}:8335", None, [DIGEST], 8, nproc, load, 0, 64 << 30, nproc,
                           PRIORITY_DEDICATED if dedicated else PRIORITY_USER))
    return out


def _cap(sv: Servant, r: int) -> int:
    avail = max(sv.num_processors - max(sv.current_load - r, 0), 0)
    return min(sv.max_tasks, avail)


def _tier(sv: Servant, r: int) -> int:
    return 0 if sv.priority == PRIORITY_DEDICATED and 2 * r < sv.num_processors else 1


def request_ips(n: int, self_frac: float, seed: int) -> list[str]:
    rng = np.random.default_rng(seed)
    ips = [f"172.16.{i >> 8}.{i & 255}" for i in rng.integers(0, 4096, n)]
    for i in np.nonzero(rng.random(n) < self_frac)[0]:
        ips[i] = f"10.77.0.{int(rng.integers(0, 10))}"
    return ips


def key_stream(d, name: str, batch: int, with_self: bool = False) -> S.Stream:
    """Heartbeats, then the long walk (and, `with_self`, the self-IP batch) offered in batches of `batch`."""
    lo, hi = CLUSTERS[name]
    ev = [("hb", 0.0, sv, 100.0) for sv in key_servants(lo, hi)]
    env = d.intern_env(DIGEST)
    queues = [request_ips(N_SELF if with_self else N_WALK, 0.1 if with_self else 0.0, seed=len(name))]
    for ips in queues:
        ip_ids = np.asarray([d.intern_ip(x) for x in ips], dtype=np.uint32)
        reqs = S._requests(d, np.full(len(ips), env, np.uint32), ip_ids, 8)
        for a in range(0, len(reqs), batch):
            ev.append(("wait", 0.001, reqs[a:a + batch]))
    ev.append(("state",))
    return S.Stream(f"keys-{name}", ev)


def model_walk(name: str, with_self: bool = False):
    """(status, servant_index, r before the grant, cap at that r) per request; the servants' final running_tasks."""
    lo, hi = CLUSTERS[name]
    svs = key_servants(lo, hi)
    ips = request_ips(N_SELF if with_self else N_WALK, 0.1 if with_self else 0.0, seed=len(name))
    own = [sv.observed_location.split(":")[0] for sv in svs]
    run = [0] * len(svs)
    status, pick, rs, caps = [], [], [], []
    for ip in ips:
        self_i, best_d, best_a, u_d, u_a = -1, -1, -1, 0.0, 0.0
        for i, sv in enumerate(svs):
            cap = _cap(sv, run[i])
            if run[i] >= cap:
                continue
            if self_i < 0 and own[i] == ip:
                self_i = i
                continue
            u = run[i] / cap
            if _tier(sv, run[i]) == 0 and (best_d < 0 or u < u_d):
                best_d, u_d = i, u
            if best_a < 0 or u < u_a:
                best_a, u_a = i, u
        i = best_d if best_d >= 0 else best_a if best_a >= 0 else self_i
        if i < 0:
            status.append(STATUS_TIMEOUT); pick.append(-1); rs.append(-1); caps.append(0)
            continue
        status.append(STATUS_GRANTED); pick.append(i); rs.append(run[i]); caps.append(_cap(svs[i], run[i]))
        run[i] += 1
    return np.asarray(status), np.asarray(pick), np.asarray(rs), np.asarray(caps), run


def check_walk(name: str) -> None:
    """The walk without self-IP requests visits slots in increasing (tier, r / cap, position), exactly; and it reaches
    the edge of its cluster: adjacent slots closer than 2^-25 (narrow / wide near 8192) or 2^-27 (16 k, where 27-bit
    floors of distinct fractions coincide -- and, for some adjacent pair, would put the higher position first)."""
    lo, hi = CLUSTERS[name]
    svs = key_servants(lo, hi)
    status, pick, rs, caps, _ = model_walk(name)
    assert (status == STATUS_GRANTED).all()
    keys = [(_tier(svs[i], r), Fraction(int(r), int(c)), int(i)) for i, r, c in zip(pick, rs, caps)]
    assert all(a < b for a, b in zip(keys, keys[1:]))
    same_tier = [(a, b) for a, b in zip(keys, keys[1:]) if a[0] == b[0] and a[1] != b[1]]
    gap = min(b[1] - a[1] for a, b in same_tier)
    merged = [(a, b) for a, b in same_tier if (a[1] * 2**27).__floor__() == (b[1] * 2**27).__floor__()]
    if hi <= 8193:
        assert gap < Fraction(1, 2**25), float(gap)
        assert not merged  # (capacities <= 8193: every pair of distinct fractions keeps distinct 27-bit floors)
    else:
        assert gap < Fraction(1, 2**27), float(gap)
        assert any(a[2] > b[2] for a, b in merged), "no adjacent pair that a 27-bit key would reorder"
