"""A window of WaitForStartingTask RPCs with 8-byte grants (yd_wait_for_starting_task_rpcs_packed,
include/ydrpcs_packed.h).  It is defined as the unpacked call, then yd_pack_grant of every grant with {next task id
before the call, stride}; every granted decision is reported, so grants_out[k] has ordinal k.  CPU part: the checkers'
packed call against that definition done by hand on twin handles, the refusals, the header's exports.  GPU part: the CUDA
call against the reference checker's packed call, against the CUDA unpacked call on twin handles (answers, exported
state, servant state, next task id) over windows on both sides of every path's threshold, its byte counts, and the
range-sharded group form (tests/shard_rpcs_packed_check.py)."""
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from rpc_packed_cases import DIGS, by_definition, cluster, ordinals_are_positions, packed, play, to_rpcs, window_rows
from yadcc_b200 import Servant, _abi, unpack_grants
from yadcc_b200 import streams as S

ROOT = Path(__file__).resolve().parent.parent
SEEDS = range(40)
REFUSED = (1 << 64) - 1


# ---- CPU: the checkers against the definition --------------------------------------------------------------------------

def test_header_is_exported_by_the_product_and_the_port_builds():
    """include/ydrpcs_packed.h is declared one-to-one in _abi.RPCS_PACKED_PROTOTYPES and exported by the CUDA library
    (required by load_library) and by every port build.  (Like ydfilter_packed.h it is not part of what ydsched.h
    requires of every library: reference checker builds made from earlier trees do not have it.)"""
    from conftest import CUDA_LIB, PORT_LIB
    from test_abi import header_symbols

    names = header_symbols("ydrpcs_packed.h")
    assert names == sorted(name for name, _, _ in _abi.RPCS_PACKED_PROTOTYPES)
    assert not set(names) & set(header_symbols())
    for lib in (CUDA_LIB, PORT_LIB, ROOT / "checkers" / "libydport_state.so", ROOT / "checkers" / "libydport_keys.so"):
        h = C.CDLL(str(lib))
        assert all(hasattr(h, name) for name in names), lib


@pytest.mark.parametrize("kind", ["port", "ref"])
@pytest.mark.parametrize("seed", SEEDS)
def test_packed_window_is_its_definition(make_dispatcher, kind, seed):
    """Seeded streams (limits at 10 000 / 10 001 ms and 30 s / 30 s + 1 ns, a digest nobody holds, prefetch-only RPCs,
    counts up to 0xFFFFFFFF, frees and ticks between windows): the port's packed call against the definition done by
    hand on a twin handle of `kind` (the port's unpacked call, or the reference's literal loops): results, packed grants
    and ids equal, and every grants_out[k] has ordinal k."""
    assert play(make_dispatcher("port"), make_dispatcher(kind), packed, by_definition, seed) >= 0


@pytest.mark.parametrize("kind", ["port", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_refusals_decide_nothing(make_dispatcher, kind):
    """cap one short of yd_rpc_expanded_requests(): (size_t)-1, *ids still written, nothing decided.  (The reference
    checker runs the reference's literal loops, which have no cap to refuse.)"""
    d = make_dispatcher(kind)
    rng = np.random.default_rng(5)
    for sv in cluster(rng):
        d.keep_servant_alive(sv, 10.0, now=0.0)
    bound = int(d._lib.yd_grant_capacity_bound(d._h))
    rpcs = to_rpcs(d, window_rows(rng, bound, 30))
    total = int(d._lib.yd_rpc_expanded_requests(d._h, rpcs.ctypes.data, len(rpcs)))
    assert total > 0
    before = (d.next_task_id(), d.servant_state().tobytes(), d.num_tasks())
    res = np.zeros(len(rpcs), dtype=_abi.RPC_RESULT_DTYPE)
    g8 = np.zeros(total, dtype=_abi.GRANT8_DTYPE)
    ids = np.zeros(1, dtype=_abi.PACKED_IDS_DTYPE)
    k = d._lib.yd_wait_for_starting_task_rpcs_packed(d._h, 0, rpcs.ctypes.data, len(rpcs), res.ctypes.data,
                                                     g8.ctypes.data, total - 1, ids.ctypes.data)
    assert k == REFUSED
    assert (int(ids[0]["first_task_id"]), int(ids[0]["stride"])) == (before[0], 1)
    assert (d.next_task_id(), d.servant_state().tobytes(), d.num_tasks()) == before
    with pytest.raises(ValueError):
        d._rpcs_packed_with(lambda h, now, r, n, out, g, cap, i: REFUSED, rpcs, 0.0)


def test_status_quirks_packed(make_dispatcher):
    """test_rpc_status_quirks' window through the packed call: 1006 / 1001 / 1004, grants a prefix, ordinals 0, 1, 2."""
    d = make_dispatcher("port")
    d.keep_servant_alive(Servant("10.6.1.1:8335", None, ["d"], 8, 8, 0, 0, 64 << 30, 3), 10.0, now=0.0)
    rpcs = np.zeros(6, dtype=_abi.RPC_WAIT_DTYPE)
    rpcs["requestor_ip"] = d.intern_ip("10.9.9.9")
    rpcs["next_keep_alive_ns"] = 15_000_000_000
    rpcs["env_id"] = [d.intern_env(x) for x in ["nope", "nope", "d", "d", "d", "d"]]
    rpcs["immediate_reqs"] = [1, 0, 2, 1, 1, 2]
    rpcs["prefetch_reqs"] = [1, 2, 0, 0, 1, 2]
    rpcs["milliseconds_to_wait"] = [0, 0, 0, 10001, 0, 0]
    res, g8, ids = d.wait_for_starting_task_rpcs_packed(rpcs, now=0.0)
    assert res["status"].tolist() == [1006, 1001, 0, 1004, 0, 1001]
    assert res["n_grants"].tolist() == [0, 0, 2, 0, 1, 0]
    assert res["first_grant"].tolist() == [0, 0, 0, 2, 2, 3]
    assert ordinals_are_positions(g8) and len(g8) == 3
    assert unpack_grants(g8, ids)["task_id"].tolist() == [0, 1, 2]


# ---- GPU ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_cuda_equals_reference_packed(make_dispatcher, seed):
    """The CUDA packed call against the reference checker's packed call on the CPU seeds: results, grants, ids.  A
    reference build made from an earlier tree has no packed call: then its definition, on the reference's unpacked
    call."""
    ref = make_dispatcher("ref")
    ref_packed = packed if hasattr(ref._lib, "yd_wait_for_starting_task_rpcs_packed") else by_definition
    assert play(make_dispatcher("cuda"), ref, packed, ref_packed, seed) >= 0


def unpacked(d, rpcs, now):
    res, g = d.wait_for_starting_task_rpcs(rpcs, now)
    return res.copy(), g.copy()


class Twins:
    """Two CUDA handles fed the same servants and windows: the packed call on `a`, the unpacked call on `b`."""

    def __init__(self, make_dispatcher):
        self.a, self.b = make_dispatcher("cuda"), make_dispatcher("cuda")
        self.windows = self.granted = 0

    def every(self, f):
        f(self.a)
        f(self.b)

    def window(self, rows_or_fn, now, *, device_bytes=None):
        """One window on both handles; checks answers, exported state, servant state and next task id.  Returns the
        packed call's (results, grants8, ids)."""
        make = rows_or_fn if callable(rows_or_fn) else (lambda d: to_rpcs(d, rows_or_fn))
        ra, rb = make(self.a), make(self.b)
        first = self.a.next_task_id()
        res, g8, ids = self.a.wait_for_starting_task_rpcs_packed(ra, now)
        stats = self.a.last_solve_stats()
        res_b, g_b = unpacked(self.b, rb, now)
        assert res.tobytes() == res_b.tobytes()
        assert (int(ids["first_task_id"]), int(ids["stride"])) == (first, 1)
        u = unpack_grants(g8, ids)
        for f in ("task_id", "servant_index", "status"):
            assert (u[f] == g_b[f]).all(), f
        assert ordinals_are_positions(g8)
        assert (self.a.servant_state() == self.b.servant_state()).all() and self.a.next_task_id() == self.b.next_task_id()
        assert self.a.export_state(now) == self.b.export_state(now)
        if device_bytes:
            assert stats["h2d_bytes"] == 32 * len(ra), stats
            assert stats["d2h_bytes"] == 16 * len(ra) + 8 * len(g8), stats
            assert stats["decisions"] == int(self.a._lib.yd_rpc_expanded_requests(self.a._h, ra.ctypes.data, len(ra)))
        self.windows += 1
        self.granted += len(g8)
        return res, g8, ids

    def free_and_tick(self, g8, ids, now):
        tid = unpack_grants(g8, ids)["task_id"][::3].tolist()
        self.every(lambda d: d.free_tasks(tid))
        self.every(lambda d: d.on_expiration_timer(now=now))


def rows(n, *, digest=0, imm=1, pre=0, ms=0, ka=10_000_000_000, ip="172.20.0.1"):
    return [(DIGS[digest], 0, ip, imm, pre, ms, ka)] * n


def small_cluster(t: Twins, seed=3):
    for sv in cluster(np.random.default_rng(seed)):
        t.every(lambda d: d.keep_servant_alive(sv, 3600.0, now=0.0))
    return int(t.a._lib.yd_grant_capacity_bound(t.a._h))


@pytest.mark.gpu
def test_twin_edge_windows(make_dispatcher):
    """Empty, all INVALID, every RPC failing, 0xFFFFFFFF counts (immediate and prefetch), kTinyMax (8) decisions and one
    more, prefetch-only; leases freed and a tick between windows."""
    t = Twins(make_dispatcher)
    bound = small_cluster(t)
    now = 1.0
    t.window([], now)
    t.window(rows(5, ms=10001) + rows(4, ka=30_000_000_001), now + 0.1)  # all INVALID
    t.window(rows(40, digest=3), now + 0.2)  # a digest nobody holds: every RPC 1006
    t.window(rows(40, digest=3, imm=0, pre=2), now + 0.3)  # ... prefetch-only: 1001
    greedy = [r for k in range(3) for r in rows(2, digest=k, imm=0xFFFFFFFF) + rows(1, digest=k, imm=0, pre=0xFFFFFFFF)]
    _, g8, ids = t.window(greedy, now + 0.4, device_bytes=True)
    assert 0 < len(g8) <= bound  # the first RPC of each digest took what its servants had
    t.window(rows(30, digest=1), now + 0.5, device_bytes=True)  # every RPC failing: the cluster is full
    t.free_and_tick(g8, ids, now + 0.6)
    t.window(rows(8, digest=1), now + 0.7)  # kTinyMax decisions: the host expansion
    t.window(rows(9, digest=1), now + 0.8, device_bytes=True)  # one more: the device path
    t.window(rows(4, digest=2, imm=1, pre=1), now + 0.9)
    t.window(rows(5, digest=2, imm=1, pre=1), now + 1.0, device_bytes=True)
    t.window(lambda d: to_rpcs(d, window_rows(np.random.default_rng(9), bound, 200)), now + 1.1, device_bytes=True)


def rpcs_from_requests(reqs: np.ndarray) -> np.ndarray:
    """One RPC per request: one immediate decision, or one prefetch decision for a prefetch request."""
    r = np.zeros(len(reqs), dtype=_abi.RPC_WAIT_DTYPE)
    r["env_id"], r["min_version"], r["requestor_ip"] = reqs["env_id"], reqs["min_version"], reqs["requestor_ip"]
    pre = (reqs["flags"] & _abi.REQ_FLAG_PREFETCH) != 0
    r["immediate_reqs"], r["prefetch_reqs"] = (~pre).astype(np.uint32), pre.astype(np.uint32)
    r["next_keep_alive_ns"] = reqs["expires_in_ns"]
    return r


@pytest.mark.gpu
def test_twin_cfg2_mod_and_large_windows(make_dispatcher):
    """cfg2-mod as 100 k one-decision RPCs; windows above the fused kernel's 262 144 decisions and above 1 M (greedy
    RPCs); 1 000 RPCs of 1 immediate + 0..16 prefetch; frees and ticks between them."""
    t = Twins(make_dispatcher)
    w = S.config2(100_000, 2000, 8, variant="mod")
    t.every(lambda d: w.register(d, now=0.0, expires_in=3600.0))
    bound = int(t.a._lib.yd_grant_capacity_bound(t.a._h))
    _, g8, ids = t.window(lambda d: rpcs_from_requests(w.build_requests(d)), 1.0, device_bytes=True)
    assert len(g8) == 100_000
    t.free_and_tick(g8, ids, 1.5)
    big = lambda d: np.concatenate([rpcs_from_requests(w.build_requests(d))] * 3)  # noqa: E731  300 k decisions
    _, g8, ids = t.window(big, 2.0, device_bytes=True)
    t.free_and_tick(g8, ids, 2.5)
    digests = w.digests

    def greedy(d):  # each RPC expands to 2 (bound + 1) decisions
        r = np.zeros(12, dtype=_abi.RPC_WAIT_DTYPE)
        r["env_id"] = [d.intern_env(digests[i % 8]) for i in range(12)]
        r["requestor_ip"] = d.intern_ip("172.30.0.1")
        r["immediate_reqs"] = r["prefetch_reqs"] = 0xFFFFFFFF
        r["next_keep_alive_ns"] = 30_000_000_000
        return r
    assert 12 * 2 * (bound + 1) > 1_000_000
    _, g8, ids = t.window(greedy, 3.0, device_bytes=True)
    t.free_and_tick(g8, ids, 3.5)
    pre = np.random.default_rng(4).integers(0, 17, 1000)

    def mixed(d):
        r = np.zeros(1000, dtype=_abi.RPC_WAIT_DTYPE)
        r["env_id"] = [d.intern_env(digests[i % 8]) for i in range(1000)]
        r["requestor_ip"] = [d.intern_ip(f"172.31.0.{i % 200}") for i in range(1000)]
        r["immediate_reqs"], r["prefetch_reqs"] = 1, pre
        r["next_keep_alive_ns"] = 15_000_000_000
        return r
    t.window(mixed, 4.0, device_bytes=True)
    assert t.windows == 4 and t.granted > 100_000


# ---- GPU: a range-sharded group (tests/shard_rpcs_packed_check.py) ------------------------------------------------------

HARNESS = ROOT / "tests" / "shard_rpcs_packed_check.py"


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_group_equals_one_handle_and_unpacked_twin(world):
    """W rank threads over the NCCL stand-in: every rank returns the same answers, equal to one checker handle's packed
    call and to the unpacked group call on a twin group; refusals (cap, capacities above 8192) on every rank."""
    from conftest import CUDA_LIB

    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "oracle" / "libydoracle.so", Path(CUDA_LIB)):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(HARNESS), "--world", str(world), "--rpcs", "24", "--seed", str(world)],
                       capture_output=True, text=True, timeout=900, env=dict(os.environ), cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_rpcs_packed") is True, msg
    assert lines[-1]["nccl"] == "fake_nccl" and not lines[-1]["torch_loaded"], msg
    cases = {c["case"]: c for c in lines[:-1] if "case" in c}
    assert cases["rpc-windows-packed"]["ok"] and cases["rpc-windows-packed"]["rpc_windows"] == 24, msg
    assert cases["rpc-windows-packed"]["device_windows"] > 5 and cases["rpc-windows-packed"]["refusals"] > 0, msg
    assert cases["refusal"]["ok"] and cases["refusal"]["refused_everywhere"], msg
