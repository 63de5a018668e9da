"""Shared builders for the packed RPC-window tests (tests/test_rpcs_packed.py, tests/shard_rpcs_packed_check.py): seeded
windows of WaitForStartingTask RPCs in the style of tests/rpc_cases.py, the packed call's definition done by hand, and a
lock-step player for twin handles."""
import numpy as np

from yadcc_b200 import PRIORITY_DEDICATED, PRIORITY_USER, STATUS_GRANTED, Servant, _abi

DIGS = [f"{i:064x}" for i in range(4)]  # DIGS[3] is held by nobody
LIMIT_MS = [0, 5000, 10000, 10001]  # milliseconds_to_wait: <= 10 s, one past it
LIMIT_KA = [15_000_000_000, 30_000_000_000, 30_000_000_001]  # next_keep_alive_ns: <= 30 s, one nanosecond past it


def cluster(rng):
    """A small mixed cluster: 5..60 servants, dedicated ones, partly filled, two versions."""
    out = []
    for i in range(int(rng.integers(5, 60))):
        envs = [DIGS[j] for j in rng.choice(3, size=int(rng.integers(1, 4)), replace=False)]
        nproc = int(rng.choice([4, 8, 16]))
        out.append(Servant(f"10.6.0.{i}:8335", None, envs, int(rng.choice([7, 8])), nproc, int(rng.integers(0, 4)), 0,
                           64 << 30, int(rng.integers(0, nproc)), PRIORITY_DEDICATED if i % 5 == 0 else PRIORITY_USER))
    return out


def window_rows(rng, bound: int, n: int | None = None):
    """One window's RPCs as rows (digest, min_version, requestor ip, immediate, prefetch, ms to wait, keep-alive ns):
    counts of 0..5 and, now and then, bound + 3 or 0xFFFFFFFF; prefetch-only RPCs; the limits on both sides; a digest
    nobody holds; requestors on servant hosts."""
    n = int(rng.integers(1, 40)) if n is None else n
    rows = []
    for _ in range(n):
        big = rng.random() < 0.08
        imm = int(rng.choice([bound + 3, 0xFFFFFFFF])) if big else int(rng.choice([0, 1, 1, 2, 5]))
        pre = int(rng.choice([0, 0, 1, 3, 0xFFFFFFFF], p=[0.4, 0.2, 0.2, 0.15, 0.05]))
        ms = int(rng.choice(LIMIT_MS, p=[0.3, 0.4, 0.2, 0.1]))
        ka = int(rng.choice(LIMIT_KA, p=[0.6, 0.3, 0.1]))
        rows.append((DIGS[int(rng.integers(0, 4))], int(rng.choice([0, 7, 8, 9])), f"10.6.0.{int(rng.integers(0, 80))}",
                     imm, pre, ms, ka))
    return rows


def to_rpcs(d, rows) -> np.ndarray:
    r = np.zeros(len(rows), dtype=_abi.RPC_WAIT_DTYPE)
    for i, (dg, mv, ip, imm, pre, ms, ka) in enumerate(rows):
        r[i] = (d.intern_env(dg), mv, d.intern_ip(ip), imm, pre, ms, ka)
    return r


def pack(g: np.ndarray, first: int) -> np.ndarray:
    """yd_pack_grant of every grant with {first, 1}."""
    g8 = np.zeros(len(g), dtype=_abi.GRANT8_DTYPE)
    g8["servant_index"] = g["servant_index"]
    ok = g["status"] == STATUS_GRANTED
    g8["status_ordinal"] = (g["status"].astype(np.uint32) << 30) | np.where(ok, g["task_id"] - np.uint64(first), 0).astype(np.uint32)
    return g8


def by_definition(d, rpcs, now):
    """The packed call's definition: the unpacked call, the grants packed with {next task id before the call, 1}."""
    first = d.next_task_id()
    res, g = d.wait_for_starting_task_rpcs(rpcs, now)
    return res.copy(), pack(g, first), (first, 1)


def packed(d, rpcs, now):
    res, g8, ids = d.wait_for_starting_task_rpcs_packed(rpcs, now)
    return res.copy(), g8.copy(), (int(ids["first_task_id"]), int(ids["stride"]))


def ordinals_are_positions(g8: np.ndarray) -> bool:
    return bool((g8["status_ordinal"] >> 30 == STATUS_GRANTED).all()
                and ((g8["status_ordinal"] & 0x3FFFFFFF) == np.arange(len(g8), dtype=np.uint32)).all())


def assert_same(a, b, what=""):
    (ra, ga, ia), (rb, gb, ib) = a, b
    assert ia == ib, (what, "ids", ia, ib)
    assert ra.tobytes() == rb.tobytes(), (what, "results")
    assert ga.tobytes() == gb.tobytes(), (what, "grants")


def play(da, db, fa, fb, seed: int, windows: int = 6, on_window=None):
    """A seeded stream on twin handles: the cluster, then windows decided by fa on da and fb on db, each followed by
    frees of half the grants and now and then a tick.  Every window's answers and the servant state and next task id
    afterwards must be equal; on_window(da, db, rpcs) may check more.  Returns the number of grants."""
    rng = np.random.default_rng(seed)
    for sv in cluster(rng):
        for d in (da, db):
            d.keep_servant_alive(sv, 10.0, now=0.0)
    bound = int(da._lib.yd_grant_capacity_bound(da._h))
    granted = 0
    for w in range(windows):
        now = 0.1 * (w + 1)
        rows = window_rows(rng, bound)
        a, b = fa(da, to_rpcs(da, rows), now), fb(db, to_rpcs(db, rows), now)
        assert_same(a, b, f"seed {seed} window {w}")
        assert ordinals_are_positions(a[1]), (seed, w)
        assert (da.servant_state() == db.servant_state()).all() and da.next_task_id() == db.next_task_id(), (seed, w)
        if on_window:
            on_window(da, db, to_rpcs(da, rows))
        granted += len(a[1])
        ids = (a[2][0] + (a[1]["status_ordinal"] & 0x3FFFFFFF).astype(np.uint64) * np.uint64(a[2][1]))[::2]
        if len(ids):
            for d in (da, db):
                d.free_tasks(ids.tolist())
        if w % 3 == 2:
            for d in (da, db):
                d.on_expiration_timer(now=now + 0.05)
    return granted
