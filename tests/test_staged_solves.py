"""The staged and the pre-filtered solves, call after call: requests decided from the handle's device-side queue
(yd_stage_requests + yd_wait_for_staged_tasks) and from the queue the filtered call compacts there
(yd_filter_and_wait_for_starting_new_tasks), compared bit for bit with the CPU restatement, and with the reference
where it is built.

  a  bench.py's own call sequence per workload: the parity head, then free, tick, packed, plain and staged per step
     (cfg4: the one-call filter), grants with absolute task ids and servant state after every call;
  b  solo, kept-lookup, flip and fuzz streams through `Replayer(staged=True)`: staged queues longer than the batch,
     staged queues decided again after frees and a tick, host calls with another array just before a staged one;
  c  filtered calls in a solo stream with survivors chosen exactly: none, 1, 3 and 8, batches at the 1024-request tile
     edges, bloom-only and dedupe-only calls, and the staged queue a filtered call leaves behind;
  d  the compaction's scan at its 8192-cell round edge (8191 / 8192 / 8193 tiles);
  e  the in-flight index's hash table at its edges: probe chains that wrap past the last slot, the capacity doubling,
     digest lengths around the 8-byte words, and one digest reported 3000 times.

The YDSCHED_DEBUG solve lines show which path each call took, so a case that stops reaching the speculative solve
fails instead of passing on another path."""
import collections
import time

import numpy as np
import pytest

from conftest import REF_LIB
from solve_lines import solves
from yadcc_b200 import STATUS_GRANTED, RunningTask, Servant, TaskDispatcher, pack_requests, unpack_grants
from yadcc_b200 import streams as S

COUNTS: collections.Counter = collections.Counter()
GIB = 1 << 30


def _lines_per_call(capfd, calls):
    """on_solve hook: the solve lines each call printed."""
    def hook(d, reqs, g):
        calls.append(solves(capfd.readouterr().err))
    return hook


def _count(modes, calls):
    for m, ls in zip(modes, calls):
        COUNTS[f"calls {m}"] += 1
        for x in ls:
            if m in ("exact", "longer", "reuse", "filter"):
                COUNTS[f"{'filtered' if m == 'filter' else 'staged'} spec {x['spec']}"] += 1
                if m != "filter":
                    COUNTS[f"staged {m} variant {x['variant']}"] += 1


# ---------------------------------------------------------------------------------------------------------------------
# a. bench.py's call sequence
# ---------------------------------------------------------------------------------------------------------------------

BENCH_STEPS = 4


def _bench_sequence(lib, name, capfd=None):
    """measure_workload's calls (bench.py) on one backend: [(what, step, grants)], [servant_state per step], [solve
    lines per call] (CUDA only)."""
    from bench import Cfg4Stages, build_workload

    w = build_workload(name)
    d = TaskDispatcher(lib)
    try:
        w.register(d, now=0.0, expires_in=3600.0)
        src = w.build_requests(d)
        stages = Cfg4Stages(d, w, len(src)) if name == "cfg4" else None
        n = len(src)
        reqs, out = d.alloc_requests(n), d.alloc_grants(n)
        reqs[...] = src
        reqs16, out8 = d.alloc_requests16(n), d.alloc_grants8(n)
        pack_requests(src, reqs16)
        use_packed = stages is None
        rec, states, lines = [], [], []
        if capfd is not None:
            capfd.readouterr()

        def one_pass(queue, now, mode, what, step):
            if stages is not None:
                g, _ = stages.one_call(reqs[: len(queue)], now, out)
            elif mode == "staged":
                d.stage_requests(queue)
                g = d.wait_for_staged_tasks(len(queue), now, out=out)
            elif mode == "packed":
                g8, ids = d.wait_for_starting_new_tasks_packed(reqs16[: len(queue)], now, out8=out8, unpack=False)
                g = unpack_grants(g8.copy(), ids)
            else:
                g = d.wait_for_starting_new_tasks(queue, now, out=out)
            g = g.copy()
            rec.append((what, step, g))
            if capfd is not None:
                lines.append(solves(capfd.readouterr().err))
            return g["task_id"][g["status"] == STATUS_GRANTED].copy()

        head = src.copy()  # (bench.py's CPU_SAMPLE is the whole 100 k queue for these workloads)
        d.free_tasks(one_pass(head, 1.5, "plain", "head-plain", -1))
        d.on_expiration_timer(now=1.6)
        if use_packed:
            d.free_tasks(one_pass(head, 1.7, "packed", "head-packed", -1))
            d.on_expiration_timer(now=1.8)
        reqs[...] = src
        prev = None
        for it in range(BENCH_STEPS):
            now = 2.0 + it
            if prev is not None:
                d.free_tasks(prev)
            d.on_expiration_timer(now=now)
            prev = one_pass(src if stages is not None else reqs, now, "packed" if use_packed else "plain",
                            "packed" if use_packed else "filter", it)
            if use_packed:
                d.free_tasks(prev)
                d.on_expiration_timer(now=now)
                prev = one_pass(reqs, now, "plain", "plain", it)
            d.free_tasks(prev)
            d.on_expiration_timer(now=now)
            prev = one_pass(src if stages is not None else reqs, now, "staged", "staged" if stages is None else "filter", it)
            states.append(d.servant_state().copy())
        return rec, states, lines
    finally:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2-mod", "cfg-self", "cfg2-random", "cfg4"])
def test_bench_sequence_equals_restatement(cuda_lib, port_lib, capfd, monkeypatch, name):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    rec, states, lines = _bench_sequence(cuda_lib, name, capfd)
    monkeypatch.delenv("YDSCHED_DEBUG")
    t0 = time.perf_counter()
    want, want_states, _ = _bench_sequence(port_lib, name)
    COUNTS["restatement seconds (a)"] += time.perf_counter() - t0
    assert [(a, b) for a, b, _ in rec] == [(a, b) for a, b, _ in want]
    for (what, step, g), (_, _, h) in zip(rec, want):
        assert g.shape == h.shape and (g == h).all(), (name, what, step, S.first_mismatch([g], [h]))
    for step, (a, b) in enumerate(zip(states, want_states)):
        assert (a == b).all(), (name, "servant_state after step", step)
    granted = [int((g["status"] == STATUS_GRANTED).sum()) for _, _, g in rec]
    assert min(granted) > 0, granted
    # every call printed one solve line (cfg4: none for the early wave, which ran before the capture)
    assert all(len(x) == 1 for x in lines), [len(x) for x in lines]
    spec = [(what, step, x[0]["spec"], x[0]["variant"]) for (what, step, _), x in zip(rec, lines)]
    if name == "cfg2-mod":  # the headline `value`: the staged solve is the speculative one from the second step on
        assert all(s == 1 and v == 4 for what, step, s, v in spec if what == "staged" and step >= 1), spec
    if name == "cfg4":
        # the filtered solve decides its compacted queue speculatively once the class set repeated, in every step; it
        # never misses.  (Not on both calls of every step: measured on an H100, the second filtered call of step 1 ran
        # without speculation, variant 2 -- a speed matter, not a wrong answer; both calls are checked above.)
        print(name, spec)
        assert all(s in (0, 1) for what, step, s, v in spec), spec
        for step in range(1, BENCH_STEPS):
            assert any(s == 1 and v == 4 for what, st, s, v in spec if st == step), (step, spec)
    for what, step, s, v in spec:
        COUNTS[f"bench {name} {what} spec {s}"] += 1


# ---------------------------------------------------------------------------------------------------------------------
# b. streams through the staged queue
# ---------------------------------------------------------------------------------------------------------------------

def _kept_streams():
    import test_kept_lookup as K
    return {"kept-shared": K._stream_shared_components, "kept-wide": K._stream_wide_components}


def _stream(name, d):
    kind, _, arg = name.partition(":")
    if kind == "solo":
        return S.solo_stream(d, int(arg))
    if kind == "kept":
        return _kept_streams()[arg](d)[0]
    if kind == "flip":
        from test_gpu_parity import _flip_stream
        return _flip_stream(d)
    return S.named_stream(f"fuzz-{arg}", d)


STREAMS = ([(f"solo:{s}", s // 3 % 2 == 1) for s in range(0, 24, 3)]
           + [(f"kept:{k}", p) for k in ("kept-shared", "kept-wide") for p in (False, True)]
           + [("flip:", p) for p in (False, True)]
           + [(f"fuzz:{s}", s % 4 == 1) for s in range(30)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,packed", STREAMS, ids=[f"{n}-{'packed' if p else 'plain'}" for n, p in STREAMS])
def test_staged_stream_equals_restatement(make_dispatcher, capfd, monkeypatch, name, packed):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    seed = sum(map(ord, name))
    capfd.readouterr()
    d = make_dispatcher("cuda")
    calls = []
    rp = S.Replayer(d, pinned=True, packed=packed, staged=True, seed=seed, on_solve=_lines_per_call(capfd, calls))
    tr = rp.run(S.with_repeats(_stream(name, d), seed))
    d.close()
    t0 = time.perf_counter()
    p = make_dispatcher("port")
    want = S.Replayer(p).run(S.with_repeats(_stream(name, p), seed))
    COUNTS["restatement seconds (b)"] += time.perf_counter() - t0
    assert S.traces_equal(tr, want), f"{name}: cuda staged vs port: " + S.first_mismatch(tr, want)
    assert len(calls) == len(rp.modes)
    _count(rp.modes, calls)
    COUNTS["stream runs"] += 1


def test_staged_stream_covers_both_outcomes():
    """Across the streams above: staged solves that the speculative solve decided (spec 1) and ones it missed and replayed
    from the staged queue (spec 2); every staged mode was used."""
    if COUNTS["stream runs"] != len(STREAMS):
        pytest.skip("runs after all of test_staged_stream_equals_restatement")
    print(dict(COUNTS))
    for key in ("staged spec 1", "staged spec 2", "calls exact", "calls longer", "calls reuse", "calls host"):
        assert COUNTS[key] > 0, (key, dict(COUNTS))


# ---------------------------------------------------------------------------------------------------------------------
# c. filtered calls in a solo stream, survivors chosen exactly
# ---------------------------------------------------------------------------------------------------------------------

CK_HIT = [f"cached-key-{i:013d}" for i in range(8)]    # in the bloom filter (24 bytes each)
CK_MISS = [f"missed-key-{i:013d}" for i in range(8)]   # not in it (checked below)
TD_RUN = [f"{0xa11 << 200 | i:064x}" for i in range(64)]  # running: in the in-flight index
TD_NEW = [f"{0xb22 << 200 | i:064x}" for i in range(64)]  # not running
OFFERED, CACHED, JOINED = 0, 1, 2


def _check_keys(port_lib):
    """The chosen keys against the restatement's bloom filter: no false positive decides a verdict."""
    d = TaskDispatcher(port_lib)
    try:
        d.bloom_reset()
        d.bloom_add(CK_HIT)
        assert d.bloom_possibly_contains(CK_HIT).all()
        assert not d.bloom_possibly_contains(CK_MISS).any()
    finally:
        d.close()


def _filter_cluster(d, n_servants=192, K=4):
    """A solo cluster (servant i holds digest i % K) with TD_RUN running on it and CK_HIT cached."""
    dgs = [f"{0x7c000000 + k:064x}" for k in range(K)]
    svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dgs[i % K]], 9, 64, 0, 256 * GIB, 200 * GIB, 24) for i in range(n_servants)]
    for sv in svs:
        d.keep_servant_alive(sv, 1e6, now=0.0)
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    ips = np.asarray([d.intern_ip(f"172.20.0.{i}") for i in range(200)], dtype=np.uint32)
    early = d.wait_for_starting_new_tasks(S._requests(d, env[np.arange(256) % K], ips[np.arange(256) % 200], 8,
                                                      expires_in_s=1e5), 0.0)
    by = {}
    for j, g in enumerate(early[: len(TD_RUN)]):
        assert g["status"] == STATUS_GRANTED
        loc = d.servant_location(int(g["servant_index"]))
        by.setdefault(loc, []).append(RunningTask(j + 1, int(g["task_id"]), loc, TD_RUN[j]))
    d.notify_servants_running_tasks(list(by.items()))
    assert d.running_index_refresh() == len(TD_RUN)
    d.bloom_reset()
    d.bloom_add(CK_HIT)
    return env, ips


def _keys(verdict, rng):
    """Cache keys and task digests (uint8 matrices) that give these verdicts."""
    n = len(verdict)
    km = TaskDispatcher._key_matrix(CK_HIT + CK_MISS)
    dm = TaskDispatcher._key_matrix(TD_RUN + TD_NEW)
    k = rng.integers(0, 8, n)
    ck = km[np.where(verdict == CACHED, k, 8 + k)]
    t = rng.integers(0, 64, n)
    td = dm[np.where(verdict == JOINED, t, np.where(verdict == CACHED, rng.integers(0, 128, n), 64 + t))]
    return ck, td


def _filter_stream(d):
    """meta["kinds"]: (kind, offered) per filtered call, in order."""
    env, ips = _filter_cluster(d)
    rng = np.random.default_rng(23)
    # the id staging of FreeTask / KeepTaskAlive at its largest size first (as in streams.solo_stream): a device buffer
    # that grows drops the kept class table, and the frees between batches would grow it now and then
    bogus = np.arange(1 << 40, (1 << 40) + (1 << 17), dtype=np.uint64)
    ev, kinds, st = [("free", bogus), ("keepalive", 0.5, bogus, 1.0)], [], {"now": 1.0}

    def reqs(n):
        return S._requests(d, env[rng.integers(0, len(env), n)], ips[rng.integers(0, len(ips), n)], 8, expires_in_s=15.0,
                           prefetch=rng.random(n) < 0.2)

    def between():
        ev.append(("state",))
        ev.append(("free_frac", int(rng.integers(1 << 30)), 0.5))
        st["now"] += 0.01
        ev.append(("tick", st["now"]))

    def filtered(kind, verdict, stages="both"):
        r = reqs(len(verdict))
        ck, td = _keys(verdict, rng)
        ev.append(("filter", st["now"], r, None if stages == "dedupe" else ck, None if stages == "bloom" else td))
        kinds.append((kind, int((verdict == OFFERED).sum()) if stages == "both" else None))
        between()
        return r

    def steady(n=1000):
        return np.where(rng.random(n) < 0.7, OFFERED, np.where(rng.random(n) < 0.6, CACHED, JOINED))

    def exactly(n, k):
        v = np.where(rng.random(n) < 0.5, CACHED, JOINED)
        v[rng.choice(n, k, replace=False)] = OFFERED
        return v

    for _ in range(5):
        filtered("steady", steady())
    filtered("kept-0", np.full(1000, CACHED))
    filtered("after-kept-0", steady())
    filtered("steady", steady())
    for k in (1, 3, 8):
        filtered(f"kept-{k}", exactly(1000, k))
    for n in (1023, 1024, 1025, 2047, 2049):
        v = steady(n)
        i = np.arange(n)
        v[(i % 1024 == 0) | (i % 1024 == 1023) | (i == n - 1)] = OFFERED
        filtered(f"n-{n}", v)
    for _ in range(3):
        filtered("steady", steady())
    for stages in ("bloom", "dedupe", "both", "bloom", "both", "dedupe"):
        filtered(f"only-{stages}" if stages != "both" else "steady", steady(), stages)
    # stage(q), filter(r), then the filtered call's survivors and a prefix of them from the staged queue
    ev.append(("wait", st["now"], reqs(900)))
    between()
    v = steady()
    r = filtered("contract", v)
    ev.append(("wait", st["now"], r[v == OFFERED]))
    between()
    ev.append(("wait", st["now"], r[v == OFFERED][:300]))
    between()
    return S.Stream("filtered-solo", ev, {"kinds": kinds})


def test_filtered_call_leaves_its_offered_requests_staged(port_lib):
    """The checkers' definition of the staged queue after a filtered call (ydsched.h): a staged replay, which decides
    the filtered call's survivors from the staged queue without staging them again, equals the plain replay."""
    _check_keys(port_lib)
    traces, modes = [], []
    for staged in (False, True):
        d = TaskDispatcher(port_lib)
        rp = S.Replayer(d, staged=staged, seed=5)
        traces.append(rp.run(_filter_stream(d)))
        modes.append(rp.modes)
        d.close()
    assert S.traces_equal(*traces), S.first_mismatch(*traces)
    assert modes[1][-2:] == ["reuse", "reuse"], modes[1]


@pytest.mark.gpu
def test_filtered_solo_stream_equals_restatement(cuda_lib, port_lib, capfd, monkeypatch):
    _check_keys(port_lib)
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    capfd.readouterr()
    d = TaskDispatcher(cuda_lib)
    calls = []
    rp = S.Replayer(d, pinned=True, staged=True, seed=9, on_solve=_lines_per_call(capfd, calls))
    stream = _filter_stream(d)
    capfd.readouterr()  # (the cluster's set-up solve)
    tr = rp.run(stream)
    d.close()
    monkeypatch.delenv("YDSCHED_DEBUG")
    wants = {}
    for kind, lib in (("port", port_lib), ("ref", str(REF_LIB))):
        if kind == "ref" and not REF_LIB.exists():
            continue
        p = TaskDispatcher(lib)
        wants[kind] = S.Replayer(p).run(_filter_stream(p))
        p.close()
    for kind, want in wants.items():
        assert S.traces_equal(tr, want), f"cuda staged vs {kind}: " + S.first_mismatch(tr, want)
    _count(rp.modes, calls)

    assert rp.modes[-2:] == ["reuse", "reuse"], rp.modes
    filt = [ls for m, ls in zip(rp.modes, calls) if m == "filter"]
    kinds = stream.meta["kinds"]
    assert len(filt) == len(kinds)
    for (kind, offered), ls in zip(kinds, filt):
        assert len(ls) == (0 if offered == 0 else 1), (kind, ls)  # (kept == 0: nothing to solve)
        if offered:
            assert ls[0]["n"] == offered and ls[0]["tiny"] == 0, (kind, ls)  # the general path from HBM, even for 1
    spec = [(k, ls[0]["spec"] if ls else None) for (k, _), ls in zip(kinds, filt)]
    assert all(s != 2 for _, s in spec), spec  # (every filtered batch has the class set of the steady ones)
    # a steady batch after one of its own size class is decided speculatively; so is the batch after a call that
    # offered nothing, which left the kept state as it was
    follow = [s for (k0, _), (k, s) in zip(spec, spec[1:]) if k in ("steady", "after-kept-0") and k0 in ("steady", "kept-0")]
    assert len(follow) >= 6 and all(s == 1 for s in follow), spec
    COUNTS["filtered spec 1 (c)"] += sum(s == 1 for _, s in spec)


# ---------------------------------------------------------------------------------------------------------------------
# d. the compaction's scan at its round edge
# ---------------------------------------------------------------------------------------------------------------------

SCAN_ROUND = 8192  # cells k_scan_u32 covers per round; the filter scans nt + 1 tile counts
SCAN_NS = (8191 * 1024, 8192 * 1024, 8192 * 1024 + 1)


def _scan_edge_calls(lib):
    d = TaskDispatcher(lib)
    try:
        env, ips = _filter_cluster(d, n_servants=512)
        n = max(SCAN_NS)
        rng = np.random.default_rng(31)
        reqs = S._requests(d, env[rng.integers(0, len(env), n)], ips[rng.integers(0, len(ips), n)], 8, expires_in_s=15.0)
        i = np.arange(n)
        tile = i // 1024
        keep = (i % 997 == 0) | ((tile == 0) & (i % 2 == 0))
        keep |= np.isin(tile, (8190, 8191, 8192)) & ((i % 4 == 0) | (i % 1024 == 1023))
        keep[-1] = True  # the one request of tile 8192
        km = TaskDispatcher._key_matrix(CK_HIT[:1] + CK_MISS[:1])
        keys = km[keep.astype(np.int64)]
        del i, tile
        out, seconds = [], []
        for k, m in enumerate(SCAN_NS):
            t0 = time.perf_counter()
            v, _, g = d.filter_and_wait_for_starting_new_tasks(reqs[:m], keys[:m], None, 2.0 + k, want_hits=False)
            seconds.append(time.perf_counter() - t0)
            g = g.copy()
            out.append((m, v.copy(), g, int(keep[:m].sum())))
            d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED])
            d.on_expiration_timer(now=2.5 + k)
        return out, seconds
    finally:
        d.close()


@pytest.mark.gpu
def test_filter_scan_round_edge(cuda_lib, port_lib):
    """8191, 8192 and 8193 tiles: nt + 1 = 8192 cells (one round), 8193 (the total in round two) and 8194 (a tile with
    survivors in round two).  About 1 % of the requests survive, in tiles 0, 8190, 8191 and 8192 and sparsely between."""
    _check_keys(port_lib)
    got, _ = _scan_edge_calls(cuda_lib)
    want, secs = _scan_edge_calls(port_lib)
    COUNTS["restatement seconds (d)"] += sum(secs)
    for (m, v, g, kept), (m2, v2, g2, _) in zip(got, want):
        assert m == m2 and (m + 1023) // 1024 + 1 in (SCAN_ROUND, SCAN_ROUND + 1, SCAN_ROUND + 2)
        assert (v == v2).all(), (m, np.nonzero(v != v2)[0][:10])
        assert len(g) == len(g2) == kept == int((v == OFFERED).sum()), (m, len(g), len(g2), kept)
        assert (g == g2).all(), (m, S.first_mismatch([g], [g2]))
        assert (g["status"] == STATUS_GRANTED).any()
    print("scan edge cases n:", [m for m, *_ in got], "restatement seconds:", [round(x, 1) for x in secs])


# ---------------------------------------------------------------------------------------------------------------------
# e. the in-flight index's hash table (running_index.cuh) at its edges
# ---------------------------------------------------------------------------------------------------------------------

M64 = (1 << 64) - 1


def rt_hash(key: bytes) -> int:
    """running_index.cuh rt_hash: 8-byte little-endian words, zero padded, through a 64-bit mix."""
    h = 0x9E3779B97F4A7C15 ^ len(key)
    for w in range(0, len(key), 8):
        h ^= int.from_bytes(key[w: w + 8].ljust(8, b"\0"), "little")
        h = (h * 0xFF51AFD7ED558CCD) & M64
        h ^= h >> 32
    h = (h * 0xC4CEB9FE1A85EC53) & M64
    return h ^ (h >> 29)


def _table_mask(entries: int) -> int:
    cap = 1024
    while cap < 2 * entries:  # (load factor <= 0.5, ydsched.cu yd_running_index_refresh)
        cap <<= 1
    return cap - 1


def _homed(mask: int, k: int, length: int = 64, tag: str = "") -> list[str]:
    """k digests of `length` (>= 7) characters whose home slot is the table's last slot (`mask`)."""
    out, c = [], 0
    while len(out) < k:
        s = f"{c:x}-{tag}".rjust(length, "e")[:length]
        if (rt_hash(s.encode()) & mask) == mask and s not in out:
            out.append(s)
        c += 1
    return out


def _report(d, digests: list[str], n_servants: int = 200) -> None:
    """Heartbeats, one grant per digest, each reported as running with that digest, then a refresh."""
    from running_index_cases import _servant

    for i in range(n_servants):
        d.keep_servant_alive(_servant(i), 100, now=0.0)
    g = d.wait_for_starting_new_tasks(d.make_requests(len(digests), "d" * 64, "10.9.9.9", 0, expires_in=300), 0.0)
    assert (g["status"] == STATUS_GRANTED).all()
    by = {}
    for j, (t, s) in enumerate(zip(g, digests)):
        loc = d.servant_location(int(t["servant_index"]))
        by.setdefault(loc, []).append(RunningTask(j + 1, int(t["task_id"]), loc, s))
    d.notify_servants_running_tasks(list(by.items()))
    assert d.running_index_refresh() == len(digests)


def _index_cases():
    """(case, snapshot digests, query key lists)."""
    rng = np.random.default_rng(3)
    cases = []
    for n in (511, 512, 513):
        mask = _table_mask(n)
        wrap = _homed(mask, 24, tag=f"w{n}-")  # a run of 24 digests from the last slot on: the chain wraps to slot 0
        absent = _homed(mask, 8, tag=f"a{n}-")  # not reported: their probes walk the wrapped run to its end
        rest = [rng.bytes(32).hex() for _ in range(n - len(wrap))]
        snap = rest[: len(rest) // 2] + wrap + rest[len(rest) // 2:]
        cases.append((f"size-{n}", snap, [snap + absent + [rng.bytes(32).hex() for _ in range(50)]]))
    lengths = (0, 1, 7, 8, 9, 17, 63, 64, 65)
    mask = _table_mask(60)
    snap = []
    for ln in lengths:
        if ln == 0:
            snap.append("")
        elif ln < 7:
            snap += [f"{j:x}".rjust(ln, "0") for j in (1, 2)]
        else:
            snap += _homed(mask, 3, ln, tag=f"L{ln}") + [rng.bytes(40).hex()[:ln] for _ in range(2)]
    queries = []
    for ln in lengths:  # every digest cut or padded to each key length: equal keys only where the lengths agree
        queries.append([s[:ln].ljust(ln, "e") for s in snap])
    cases.append(("lengths", snap, queries))
    one = f"{0xc0ffee:064x}"
    cases.append(("3000-reports", [one] * 3000, [[one] * 100 + [rng.bytes(32).hex() for _ in range(50)]]))
    return cases


def _index_answers(lib, case):
    name, snap, queries = case
    d = TaskDispatcher(lib)
    try:
        _report(d, snap)
        out = [np.asarray([d.running_index_size()], dtype=np.uint64)]
        for q in queries:
            ln = len(q[0])
            m = np.frombuffer("".join(q).encode(), dtype=np.uint8).reshape(len(q), ln) if ln else np.zeros((len(q), 0), np.uint8)
            hits = d.find_running_tasks(m)
            out.append(hits)
            ent = [d.running_index_entry(int(i)) for i in hits["snapshot_index"][hits["found"] == 1]]
            out.append(np.asarray([(e.servant_task_id, e.task_grant_id) for e in ent], dtype=np.uint64).reshape(-1, 2))
            out.append(np.asarray([e.task_digest for e in ent], dtype="U80"))
        snapshot = [t.task_digest for t in d.get_running_tasks()]
        return out, snapshot
    finally:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", _index_cases(), ids=lambda c: c[0])
def test_running_index_edges_equal_restatement(cuda_lib, port_lib, case):
    got, snapshot = _index_answers(cuda_lib, case)
    want, _ = _index_answers(port_lib, case)
    assert S.traces_equal(got, want), f"{case[0]}: " + S.first_mismatch(got, want)
    name, snap, queries = case
    hits = got[1]
    # the restatement's own rule, checked once more here: a reported digest is found at its LAST snapshot entry
    for key, h in zip(queries[0], hits):
        same = [i for i, s in enumerate(snapshot) if s == key]
        assert h["found"] == bool(same) and (not same or h["snapshot_index"] == same[-1]), (name, key)
    if name.startswith("size-"):
        assert all(h["found"] for h in hits[: len(snap)])
