"""The packed pre-filtered solve (yd_filter_and_wait_for_starting_new_tasks_packed): 16-byte requests and 32-byte binary
digests up, 8-byte grants down.  It is defined as the unpacked call on the unpacked requests and the hex-expanded keys,
then yd_pack_grant with the batch's ids.  CPU part: the checkers' implementation against that definition, done here by
hand, and the Python helpers.  GPU part: the CUDA call against the reference checker's and against the CUDA unpacked call
on twin handles, the staged queue it leaves, its byte counts, and the range-sharded group form
(tests/shard_filter_packed_check.py)."""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from yadcc_b200 import RunningTask, STATUS_GRANTED, _abi, binary_digests, pack_requests, unpack_grants
from yadcc_b200 import streams as S

ROOT = Path(__file__).resolve().parent.parent
PREFIX = "yadcc-cxx2-entry-"


def hexkeys(d: np.ndarray, cache: bool) -> list[str]:
    return [(PREFIX if cache else "") + bytes(r).hex() for r in d]


def setup(d, n, n_servants=64, tu=400, seed=11, max_tasks=16, early=100):
    """config2-mod's cluster, a bloom filter over every third TU's cache key, and an in-flight index over the digests of
    `early` granted requests.  Returns (reqs, cache digests, task digests) of an n-request trace over `tu` TUs."""
    rng = np.random.default_rng(seed)
    cd_tu = np.frombuffer(rng.bytes(32 * tu), np.uint8).reshape(tu, 32)
    td_tu = np.frombuffer(rng.bytes(32 * tu), np.uint8).reshape(tu, 32)
    w = S.config2(n, n_servants, 4, variant="mod", max_tasks=max_tasks)
    w.register(d)
    d.bloom_reset()
    d.bloom_add(hexkeys(cd_tu[::3], True))
    reqs = w.build_requests(d)
    reqs["expires_in_ns"] = (reqs["expires_in_ns"] // 1_000_000) * 1_000_000
    g = d.wait_for_starting_new_tasks(reqs[:early].copy(), 0.25)
    locs = [d.servant_location(i) for i in range(n_servants)]
    by = {}
    for j, gr in enumerate(g):
        if gr["status"] == STATUS_GRANTED:
            si = int(gr["servant_index"])
            by.setdefault(si, []).append(RunningTask(j + 1, int(gr["task_id"]), locs[si], bytes(td_tu[(tu - 1 - j) % tu]).hex()))
    d.notify_servants_running_tasks([(locs[si], ts) for si, ts in sorted(by.items())])
    d.running_index_refresh()
    t = np.arange(n) % tu
    return reqs, np.ascontiguousarray(cd_tu[t]), np.ascontiguousarray(td_tu[t])


def by_definition(d, reqs16, cd, td, now, hits=True):
    """The packed call's definition: the unpacked call with the hex keys, the grants packed with the batch's ids."""
    first = d.next_task_id()
    reqs = np.zeros(len(reqs16), dtype=_abi.REQ_DTYPE)
    reqs["env_id"], reqs["min_version"], reqs["requestor_ip"] = reqs16["env_id"], reqs16["min_version"], reqs16["requestor_ip"]
    reqs["flags"] = np.where(reqs16["lease"] & _abi.LEASE_PREFETCH, _abi.REQ_FLAG_PREFETCH, 0)
    reqs["expires_in_ns"] = (reqs16["lease"] & 0x7FFFFFFF).astype(np.int64) * 1_000_000
    v, h, g = d.filter_and_wait_for_starting_new_tasks(reqs, None if cd is None else hexkeys(cd, True),
                                                       None if td is None else hexkeys(td, False), now, want_hits=hits)
    g8 = np.zeros(len(g), dtype=_abi.GRANT8_DTYPE)
    g8["servant_index"] = g["servant_index"]
    ok = g["status"] == STATUS_GRANTED
    g8["status_ordinal"] = (g["status"].astype(np.uint32) << 30) | np.where(ok, g["task_id"] - np.uint64(first), 0).astype(np.uint32)
    return v.copy(), None if h is None else h.copy(), g8, (first, 1)


def packed(d, reqs16, cd, td, now, hits=True):
    v, h, g8, ids = d.filter_and_wait_for_starting_new_tasks_packed(reqs16, cd, td, now, hits)
    return v.copy(), None if h is None else h.copy(), g8.copy(), (int(ids["first_task_id"]), int(ids["stride"]))


def same(a, b, what=""):
    for x, y, name in zip(a, b, ("verdicts", "hits", "grants", "ids")):
        if x is None or y is None:
            assert x is None and y is None, (what, name)
        elif isinstance(x, tuple):
            assert x == y, (what, name, x, y)
        else:
            assert x.shape == y.shape and (x == y).all(), (what, name)


STAGES = {"both": (True, True), "cache": (True, False), "dedupe": (False, True), "none": (False, False)}


def pick(cd, td, stages):
    c, t = STAGES[stages]
    return (cd if c else None), (td if t else None)


# ---- CPU: the checkers against the definition ---------------------------------------------------------------------------
# The packed call runs on the port (built from source with every build); the definition's unpacked call runs on the port
# and on the reference build, which has exported it all along.


def test_prefilter_packed_struct():
    assert C.sizeof(_abi.yd_prefilter_packed) == 16


def test_packed_header_is_exported_by_the_product_and_the_port_builds():
    """include/ydfilter_packed.h is declared one-to-one in _abi.FILTER_PACKED_PROTOTYPES, and exported by the CUDA
    library (required by load_library) and by every port build."""
    from conftest import CUDA_LIB, PORT_LIB
    from test_abi import header_symbols

    names = header_symbols("ydfilter_packed.h")
    assert names == sorted(name for name, _, _ in _abi.FILTER_PACKED_PROTOTYPES)
    assert not set(names) & set(header_symbols())  # (not part of what ydsched.h requires of every library)
    for lib in (CUDA_LIB, PORT_LIB, ROOT / "checkers" / "libydport_state.so", ROOT / "checkers" / "libydport_keys.so"):
        h = C.CDLL(str(lib))
        assert all(hasattr(h, name) for name in names), lib


@pytest.mark.parametrize("kind", ["port", "ref"])
@pytest.mark.parametrize("stages", list(STAGES))
def test_packed_prefiltered_solve_is_its_definition(make_dispatcher, kind, stages):
    """The fixture of test_prefiltered_solve_is_the_three_calls_in_order: verdicts, hits, grants, ids, and the staged
    queue afterwards decided again."""
    out = []
    for d_kind, fn in (("port", packed), (kind, by_definition)):
        d = make_dispatcher(d_kind)
        reqs, cd, td = setup(d, 2000)
        r16 = pack_requests(reqs)
        cdx, tdx = pick(cd, td, stages)
        res = fn(d, r16, cdx, tdx, 0.5)
        again = d.wait_for_staged_tasks(len(res[2]), 0.75).copy() if len(res[2]) else None
        out.append((res, again, d.servant_state()["running_tasks"].copy(), d.next_task_id()))
    same(out[0][0], out[1][0], stages)
    assert (out[0][2] == out[1][2]).all() and out[0][3] == out[1][3]
    if out[0][1] is not None:
        assert (out[0][1] == out[1][1]).all()
    v = out[0][0][0]
    assert (v == _abi.FILTER_OFFERED).sum() == len(out[0][0][2])
    if stages == "both":
        assert (v == _abi.FILTER_CACHE_HIT).any() and (v == _abi.FILTER_JOINED).any()
        assert (out[0][0][2]["status_ordinal"] >> 30 == STATUS_GRANTED).any()


def fuzz_calls(d, fn, seed, calls=12, churn=False):
    """Calls with prefetch leases, requestors on servant hosts (self-IP), frees and expiry between them; with `churn`,
    servants changing load, leaving (their heartbeats stop) and coming back between the calls."""
    rng = np.random.default_rng(seed)
    reqs, cd, td = setup(d, 600, n_servants=24, tu=60, seed=seed, max_tasks=6, early=40)
    hosts = [d.servant_location(i).split(":")[0] for i in range(24)]
    self_ips = np.asarray([d.intern_ip(h) for h in hosts], dtype=np.uint32)
    personalities = [d.servant_personality(i) for i in range(24)]  # (a servant that expires leaves the registry)
    out, held = [], []
    for k in range(calls):
        n = int(rng.choice([1, 7, 60, 300, 600]))
        idx = rng.integers(0, len(reqs), n)
        r = reqs[idx].copy()
        r["flags"] = (rng.random(n) < 0.3).astype(np.uint32) * _abi.REQ_FLAG_PREFETCH
        r["expires_in_ns"] = rng.integers(0, 30_000, n) * 1_000_000
        own = rng.random(n) < 0.25
        r["requestor_ip"][own] = self_ips[rng.integers(0, len(self_ips), int(own.sum()))]
        stages = list(STAGES)[k % 4]
        cdx, tdx = pick(np.ascontiguousarray(cd[idx]), np.ascontiguousarray(td[idx]), stages)
        now = 1.0 + 0.5 * k
        res = fn(d, pack_requests(r), cdx, tdx, now, hits=bool(k % 2))
        g = unpack_grants(res[2], np.asarray(res[3], dtype=np.uint64).view(_abi.PACKED_IDS_DTYPE)[0]) if len(res[2]) else res[2]
        if len(res[2]):
            held += g["task_id"][g["status"] == STATUS_GRANTED].tolist()
        if held and k % 3 == 2:
            d.free_tasks(np.asarray(held[::2], dtype=np.uint64))
            held = held[1::2]
        if churn:
            for i in range(k % 3, 24, 3):
                sv = personalities[i]
                sv.current_load = int(rng.integers(0, sv.num_processors + 1))
                d.keep_servant_alive(sv, 0.2 if k % 4 == 1 else 30.0, now=now + 0.05)
        d.on_expiration_timer(now=now + 0.3)
        out.append(res)
    return out


@pytest.mark.parametrize("kind", ["port", "ref"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_packed_prefiltered_fuzz_is_its_definition(make_dispatcher, kind, seed):
    a = fuzz_calls(make_dispatcher("port"), packed, seed)
    b = fuzz_calls(make_dispatcher(kind), by_definition, seed)
    for k, (x, y) in enumerate(zip(a, b)):
        same(x, y, k)
    assert any(len(x[2]) and (x[2]["status_ordinal"] >> 30 == STATUS_GRANTED).any() for x in a)


def nibble_digests():
    """Every nibble value in every position, and the all-0x00 / all-0xff records."""
    rows = [np.zeros(32, np.uint8), np.full(32, 0xFF, np.uint8)]
    for v in range(16):
        rows.append(np.full(32, v * 17, np.uint8))  # both nibbles v
        rows.append(((np.arange(32) + v) % 16 * 16 + (15 - (np.arange(32) + v) % 16)).astype(np.uint8))
    return np.ascontiguousarray(np.stack(rows))


def nibble_verdicts(d, packed_form, d_cache, d_task):
    """Half the records in the bloom filter and half in the in-flight index (by their hex keys), then one call."""
    n = len(d_cache)
    w = S.config2(n, 8, 2, variant="mod")
    w.register(d)
    reqs = w.build_requests(d)
    reqs["expires_in_ns"] = 10_000_000_000
    d.bloom_reset(1 << 12, 3)
    d.bloom_add(hexkeys(d_cache[::2], True))
    g = d.wait_for_starting_new_tasks(reqs[:8].copy(), 0.1)
    loc = [d.servant_location(i) for i in range(8)]
    by = {}
    for j, gr in enumerate(g):
        if gr["status"] == STATUS_GRANTED:
            si = int(gr["servant_index"])
            by.setdefault(si, []).append(RunningTask(j + 1, int(gr["task_id"]), loc[si], bytes(d_task[1 + 2 * j]).hex()))
    d.notify_servants_running_tasks([(loc[si], ts) for si, ts in sorted(by.items())])
    d.running_index_refresh()
    fn = packed if packed_form else by_definition
    return fn(d, pack_requests(reqs), d_cache, d_task, 0.5)


@pytest.mark.parametrize("kind", ["port", "ref"])
def test_every_nibble_gives_the_hex_keys_verdicts(make_dispatcher, kind):
    dg = nibble_digests()
    dt = np.ascontiguousarray(dg[::-1])
    a = nibble_verdicts(make_dispatcher("port"), True, dg, dt)
    b = nibble_verdicts(make_dispatcher(kind), False, dg, dt)
    same(a, b)
    assert (a[0] == _abi.FILTER_CACHE_HIT).any() and (a[0] == _abi.FILTER_JOINED).any()


def test_packed_prefiltered_edges(make_dispatcher):
    d = make_dispatcher("port")
    reqs, cd, td = setup(d, 400)
    r16 = pack_requests(reqs)
    before = d.next_task_id()
    # nothing filtered, n = 0
    v, h, g8, ids = d.filter_and_wait_for_starting_new_tasks_packed(r16[:0], cd[:0], td[:0], 0.3, True)
    assert len(v) == len(g8) == 0 and int(ids["first_task_id"]) == before and int(ids["stride"]) == 1
    # n = 1, both stages NULL: the one request is offered
    v, h, g8, ids = d.filter_and_wait_for_starting_new_tasks_packed(r16[200:201].copy(), None, None, 0.4, True)
    assert v.tolist() == [0] and len(g8) == 1 and not h["found"].any() and int(ids["first_task_id"]) == before
    # everything filtered out: only cached TUs, the cache stage alone
    cached = np.ascontiguousarray(np.repeat(cd[:1], 50, axis=0))
    nxt = d.next_task_id()
    v, h, g8, ids = d.filter_and_wait_for_starting_new_tasks_packed(np.ascontiguousarray(r16[:50]), cached, None, 0.5)
    assert (v == _abi.FILTER_CACHE_HIT).all() and len(g8) == 0 and h is None
    assert int(ids["first_task_id"]) == nxt == d.next_task_id()
    # the dedupe stage alone
    a = packed(d, np.ascontiguousarray(r16[280:]), None, np.ascontiguousarray(td[280:]), 0.6)  # (TUs 280 ..: some run)
    assert (a[0] != _abi.FILTER_CACHE_HIT).all() and (a[0] == _abi.FILTER_JOINED).any()


def test_binary_digests_helper():
    rng = np.random.default_rng(0)
    raw = np.frombuffer(rng.bytes(32 * 5), np.uint8).reshape(5, 32)
    assert (binary_digests(hexkeys(raw, False)) == raw).all()
    assert (binary_digests(hexkeys(raw, True)) == raw).all()
    assert (binary_digests(hexkeys(nibble_digests(), True)) == nibble_digests()).all()
    for bad in (["ab" * 31], [PREFIX.upper() + "00" * 32], ["AB" * 32], ["zz" * 32]):
        with pytest.raises(ValueError):
            binary_digests(bad)


# ---- GPU: the CUDA call ----------------------------------------------------------------------------------------------------


def checker(make_dispatcher):
    """The reference build if it exports the packed call (builds of this tree do), else the port."""
    from conftest import REF_LIB

    if REF_LIB.exists() and hasattr(C.CDLL(str(REF_LIB)), "yd_filter_and_wait_for_starting_new_tasks_packed"):
        return make_dispatcher("ref")
    return make_dispatcher("port")


def cfg4_setup(d, n):
    """The test_cfg4_prefiltered_solve_in_one_call set-up with binary digests."""
    rng = np.random.default_rng(4)
    tu = 6124
    cd_tu = np.frombuffer(np.random.default_rng(46).bytes(32 * tu), np.uint8).reshape(tu, 32)
    td_tu = np.frombuffer(np.random.default_rng(11).bytes(32 * tu), np.uint8).reshape(tu, 32)
    cached = cd_tu[rng.random(tu) < 0.3]
    w = S.config2(n, 2000, 8, variant="mod")
    w.register(d)
    d.bloom_reset()
    d.bloom_add(hexkeys(cached, True))
    reqs = w.build_requests(d)
    reqs["expires_in_ns"] = (reqs["expires_in_ns"] // 1_000_000) * 1_000_000
    early = d.wait_for_starting_new_tasks(reqs[:1500].copy(), 0.25)
    locs = [d.servant_location(i) for i in range(2000)]
    by = {}
    for j, gr in enumerate(early):
        si = int(gr["servant_index"])
        by.setdefault(si, []).append(RunningTask(j + 1, int(gr["task_id"]), locs[si], bytes(td_tu[5000 - j]).hex()))
    d.notify_servants_running_tasks([(locs[si], ts) for si, ts in sorted(by.items())])
    d.running_index_refresh()
    t = np.arange(n) % tu
    return pack_requests(reqs), np.ascontiguousarray(cd_tu[t]), np.ascontiguousarray(td_tu[t])


def unpack(res):
    return unpack_grants(res[2], np.asarray(res[3], dtype=np.uint64).view(_abi.PACKED_IDS_DTYPE)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("stages", list(STAGES))
def test_cfg4_packed_equals_checker_and_unpacked(make_dispatcher, stages):
    """100 k requests: the CUDA packed call equals the checker's and the definition on the reference build, its grants
    unpacked equal the CUDA unpacked call's on a twin handle, and the staged queue it leaves decides like the unpacked
    call's."""
    from conftest import REF_LIB

    res = []
    runs = [("cuda", packed), ("check", packed), ("cuda", by_definition)] + ([("ref", by_definition)] if REF_LIB.exists() else [])
    for kind, fn in runs:
        d = checker(make_dispatcher) if kind == "check" else make_dispatcher(kind)
        r16, cd, td = cfg4_setup(d, 100_000)
        cdx, tdx = pick(cd, td, stages)
        out = fn(d, r16, cdx, tdx, 0.5)
        again = d.wait_for_staged_tasks(len(out[2]), 0.75).copy() if len(out[2]) else None
        res.append((out, again, d.servant_state()["running_tasks"].copy()))
    same(res[0][0], res[1][0], "cuda vs checker")
    for y in res[2:]:
        same(res[0][0], y[0], "cuda packed vs a definition")
    for y in res[1:]:
        x = res[0]
        assert (x[2] == y[2]).all()
        assert (x[1] is None) == (y[1] is None) and (x[1] is None or (x[1] == y[1]).all())
    v = res[0][0][0]
    if stages == "both":
        assert 0.2 < (v == _abi.FILTER_CACHE_HIT).mean() < 0.4 and (v == _abi.FILTER_JOINED).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1023, 1024, 1025, 1, 5000])
def test_packed_compaction_tile_edges(make_dispatcher, n):
    res = []
    for kind, fn in (("cuda", packed), ("check", packed), ("cuda", by_definition)):
        d = checker(make_dispatcher) if kind == "check" else make_dispatcher(kind)
        reqs, cd, td = setup(d, max(n, 2000))
        res.append(fn(d, pack_requests(reqs[:n].copy()), cd[:n].copy(), td[:n].copy(), 0.5))
    same(res[0], res[1], "cuda vs checker")
    same(res[0], res[2], "cuda packed vs cuda definition")


@pytest.mark.gpu
def test_packed_scan_round_edge(make_dispatcher):
    """8191, 8192 and 8193 tiles of 1024 requests (the compaction scan's round edge, as in test_staged_solves.py): the
    packed call against the CUDA unpacked call on a twin handle (which test_staged_solves.py checks against the
    checker at these sizes)."""
    ns = (8191 * 1024, 8192 * 1024, 8192 * 1024 + 1)
    out = []
    for fn in (packed, by_definition):
        d = make_dispatcher("cuda")
        w = S.config2(max(ns), 512, 8, variant="mod")
        w.register(d)
        reqs = w.build_requests(d)
        reqs["expires_in_ns"] = 15_000_000_000
        r16 = pack_requests(reqs)
        del reqs
        hit, miss = np.full(32, 0x5A, np.uint8), np.full(32, 0xA5, np.uint8)
        d.bloom_reset()
        d.bloom_add(hexkeys(hit[None], True))
        i = np.arange(max(ns))
        tile = i // 1024
        keep = (i % 997 == 0) | ((tile == 0) & (i % 2 == 0))
        keep |= np.isin(tile, (8190, 8191, 8192)) & ((i % 4 == 0) | (i % 1024 == 1023))
        keep[-1] = True
        cd = np.ascontiguousarray(np.where(keep[:, None], miss, hit).astype(np.uint8))
        del i, tile
        res = []
        for k, m in enumerate(ns):
            r = fn(d, r16[:m], cd[:m], None, 2.0 + k, hits=False)
            assert len(r[2]) == int(keep[:m].sum())
            res.append(r)
            g = unpack(r)
            d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED])
            d.on_expiration_timer(now=2.5 + k)
        out.append(res)
        d.close()
    for x, y in zip(*out):
        same(x, y)
        assert (x[2]["status_ordinal"] >> 30 == STATUS_GRANTED).any()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_packed_fuzz_equals_checker(make_dispatcher, seed):
    """The fuzz streams of the CPU test, with servant churn after them: CUDA packed, checker packed, CUDA definition."""
    runs = [fuzz_calls(make_dispatcher("cuda"), packed, seed, 16, True),
            fuzz_calls(checker(make_dispatcher), packed, seed, 16, True),
            fuzz_calls(make_dispatcher("cuda"), by_definition, seed, 16, True)]
    for k, (a, b, c) in enumerate(zip(*runs)):
        same(a, b, ("checker", k))
        same(a, c, ("definition", k))


@pytest.mark.gpu
def test_every_nibble_on_the_gpu(make_dispatcher):
    dg = nibble_digests()
    dt = np.ascontiguousarray(dg[::-1])
    a = nibble_verdicts(make_dispatcher("cuda"), True, dg, dt)
    b = nibble_verdicts(make_dispatcher("cuda"), False, dg, dt)
    c = nibble_verdicts(checker(make_dispatcher), True, dg, dt)
    same(a, b)
    same(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("stages", list(STAGES))
def test_packed_byte_counts(make_dispatcher, stages):
    """Against the unpacked call on a twin handle: 8 n fewer bytes up for the requests, 49 n for the cache keys, 32 n
    for the task digests; 8 fewer down per offered request."""
    st = []
    for fn in (packed, by_definition):
        d = make_dispatcher("cuda")
        reqs, cd, td = setup(d, 20_000)
        cdx, tdx = pick(cd, td, stages)
        r = fn(d, pack_requests(reqs), cdx, tdx, 0.5, hits=False)
        st.append((d.last_solve_stats(), len(r[2])))
    (a, k), (b, k2) = st
    n = 20_000
    c, t = STAGES[stages]
    assert k == k2 > 0
    assert b["h2d_bytes"] - a["h2d_bytes"] == 8 * n + (49 * n if c else 0) + (32 * n if t else 0), (a, b)
    assert b["d2h_bytes"] - a["d2h_bytes"] == 8 * k, (a, b)


# ---- GPU: the range-sharded group ------------------------------------------------------------------------------------------


def _group(*args, timeout=1200):
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "checkers" / "libydport_keys.so",
              ROOT / "yadcc_b200" / "libydsched.so"):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "shard_filter_packed_check.py"), *args], capture_output=True,
                       text=True, timeout=timeout, cwd=ROOT)
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1].get("shard_filter_packed") is True, msg
    return [x for x in lines[:-1] if "case" in x], msg


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_group_packed_equals_one_handle(world):
    """W ranks over the NCCL stand-in: every rank's verdicts, hits, packed grants and ids against one checker handle's
    packed call on the concatenated queue, and unpacked against its unpacked call; empty and wholly filtered ranges,
    the sequential fallback, the staged queue decided again, and the refusal of capacities above 8192."""
    cases, msg = _group("--world", str(world), "--fuzz", "6", "--seed", str(world))
    assert len(cases) == 2 and all(c["ok"] for c in cases), msg
    c = cases[0]
    assert c["calls"] == 4 * 6 and c["redecided"] == c["calls"] and c["offered"] > 0 and c["all_filtered"] > 0, msg
    if world > 1:
        assert c["empty_ranges"] > 0 and c["filtered_ranges"] > 0, msg
    assert cases[1]["case"] == "refusal" and cases[1]["refused_everywhere"], msg


@pytest.mark.gpu
def test_group_packed_real_nccl_one_rank():
    cases, msg = _group("--real-nccl", "--world", "1", "--fuzz", "3", "--seed", "9")
    assert cases and all(c["ok"] for c in cases), msg
