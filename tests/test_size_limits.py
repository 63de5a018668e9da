"""Both sides of every size limit that picks a solve path (ydsched.cu WaitImpl / EnqueueSolve), each against the CPU
restatement (and the reference where it is built): statuses, task ids, servant indices, servant_state() and the task
counters.  Every case reads the YDSCHED_DEBUG line of its solves and asserts that it ran the side it names, so a
case that drifts onto the common path fails instead of passing there.

Large clusters get small batches and large batches get few servants: the checkers decide in O(servants) per request.
"""
import functools

import numpy as np
import pytest

import key_cases as K
from conftest import REF_LIB
from solve_lines import solves as _solves
from yadcc_b200 import PRIORITY_DEDICATED, PRIORITY_USER, STATUS_GRANTED, Servant
from yadcc_b200 import streams as S
from yadcc_b200._abi import STATUS_ENVIRONMENT_NOT_FOUND

pytestmark = pytest.mark.gpu

GiB = 1 << 30
STATIC_SLOT_LIMIT = 1 << 26  # kStaticSlotLimit
THREE_PASS_N = (1 << 21) + 1  # nb = NextPow2(N) / 1024 > 2048
FUSED_MAX_N = 262144          # fused_max_nb


def _checkers():
    return ("port", "ref") if REF_LIB.exists() else ("port",)


@functools.lru_cache(maxsize=None)
def _oracle(case: str, kind: str):
    """A checker's trace of a named case (it does not depend on the CUDA-side options, so it is computed once)."""
    from conftest import _ensure_port
    from yadcc_b200 import TaskDispatcher

    d = TaskDispatcher(str(_ensure_port()) if kind == "port" else str(REF_LIB))
    try:
        return S.Replayer(d, batch_heartbeats=True).run(CASES[case](d))
    finally:
        d.close()


def _cuda(make_dispatcher, capfd, case, *, packed=False, graphs=True, pinned=True, stream=None, **kw):
    capfd.readouterr()
    d = make_dispatcher("cuda", graphs=graphs, **kw)
    tr = S.Replayer(d, pinned=pinned, packed=packed, batch_heartbeats=True).run((stream or CASES[case])(d))
    d.close()
    return tr, _solves(capfd.readouterr().err)


def _check(case, tr, checkers=None):
    for kind in checkers or _checkers():
        want = _oracle(case, kind)
        assert S.traces_equal(tr, want), f"cuda vs {kind}: " + S.first_mismatch(tr, want)


@pytest.fixture(autouse=True)
def _debug_line(monkeypatch):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")


def _hb(servants, now=0.0):
    return [("hb", now, sv, 100.0) for sv in servants]


# ---- kStaticSlotLimit: the kept slot order against the per-solve table ------------------------------------------------

def _slot_limit_case(n_servants: int, cap: int, extra: int):
    """n_servants x (cap + 1) slots, `extra` more on servant 0: a few thousand requests per solve, frees between the
    solves (rows of the per-solve table start at different running_tasks), then heartbeats that move servant 0 across
    the limit and back."""
    def build(d):
        rng = np.random.default_rng(cap + extra)
        dg = ["a1" * 32, "b2" * 32]
        svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[i % 2]], 8, cap, int(rng.integers(0, cap)) if i % 5 == 0 else 0,
                       0, 64 * GiB, cap, PRIORITY_DEDICATED if i % 11 == 0 else PRIORITY_USER) for i in range(n_servants)]
        svs[0] = Servant(svs[0].observed_location, None, [dg[0]], 8, cap + extra, 0, 0, 64 * GiB, cap + extra)
        env = np.asarray([d.intern_env(x) for x in dg + ["c3" * 32]], dtype=np.uint32)
        ips = np.asarray([d.intern_ip(f"172.16.0.{i}") for i in range(64)], dtype=np.uint32)
        ev = _hb(svs)
        now = 0.001

        def solve(n=3000):
            nonlocal now
            e = env[np.where(rng.random(n) < 0.01, 2, rng.integers(0, 2, n))]
            ev.append(("wait", now, S._requests(d, e, ips[rng.integers(0, 64, n)], 8)))
            ev.append(("state",))
            ev.append(("free_frac", int(rng.integers(1 << 30)), 0.5))
            now += 0.01

        for _ in range(3):
            solve()
        for nproc in (cap + 1 - extra, cap + extra):  # across the limit, then back
            ev += _hb([Servant(svs[0].observed_location, None, [dg[0]], 8, nproc, 0, 0, 64 * GiB, nproc)], now)
            solve()
            solve()
        return S.Stream("slot-limit", ev)
    return build


SLOT_LIMIT = {  # (servants, cap, extra): static bound = servants * (cap + 1) + extra
    "narrow-inside": (8192, 8191, 0), "narrow-outside": (8192, 8191, 1),
    "wide-inside": (4096, 16383, 0), "wide-outside": (4096, 16383, 1),
}


@pytest.mark.parametrize("graphs", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("case", list(SLOT_LIMIT))
def test_static_slot_limit(make_dispatcher, capfd, case, graphs):
    n, cap, extra = SLOT_LIMIT[case]
    assert n * (cap + 1) + extra == STATIC_SLOT_LIMIT + extra
    tr, solves = _cuda(make_dispatcher, capfd, "slot-" + case, graphs=graphs)
    _check("slot-" + case, tr)
    assert len(solves) == 7
    assert all(s["wide"] == case.startswith("wide") and s["variant"] == 0 and s["final"] == 1 for s in solves), solves
    static = [s["order_static"] for s in solves]
    # the first three solves are on the side the case names, the next two on the other one, the last two back again
    side = 1 if extra == 0 else 0
    assert static == [side] * 3 + [1 - side] * 2 + [side] * 2, static
    assert solves[0]["slot_b"] == (STATIC_SLOT_LIMIT if side else 1 << (n * 3001 - 1).bit_length())  # (rows clamped to n)


# ---- the three-pass grant write (k_final_count / k_final_scan / k_final_write) ------------------------------------

def _big_batch_case(n: int):
    """~300 servants, 2.4 M slots: 280 hold digest A, 20 hold digest B (B runs out: Timeouts), 3 % unknown digests,
    the last request unknown too -- so the first n-1 decisions of this queue are the n-1-request batch's."""
    def build(d):
        rng = np.random.default_rng(21)
        dg = ["d4" * 32, "e5" * 32]
        svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[0] if i % 15 else dg[1]], 8, 8000, int(rng.integers(0, 40)),
                       0, 64 * GiB, 8000, PRIORITY_DEDICATED if i % 7 == 0 else PRIORITY_USER) for i in range(300)]
        env = np.asarray([d.intern_env(x) for x in dg + ["f6" * 32]], dtype=np.uint32)
        ips = np.asarray([d.intern_ip(f"172.17.{i >> 8}.{i & 255}") for i in range(1024)], dtype=np.uint32)
        u = rng.random(THREE_PASS_N)
        e = env[np.where(u < 0.03, 2, np.where(u < 0.30, 1, 0))]
        e[-1] = env[2]
        reqs = S._requests(d, e, ips[rng.integers(0, 1024, THREE_PASS_N)], 8)
        ev = _hb(svs)
        if n == THREE_PASS_N:
            ev.append(("wait", 0.001, reqs))
        elif n == 0:  # two consecutive halves: decisions compose
            ev += [("wait", 0.001, reqs[: 1 << 20]), ("wait", 0.001, reqs[1 << 20:])]
        else:
            ev.append(("wait", 0.001, reqs[:n]))
        ev.append(("state",))
        return S.Stream("big", ev)
    return build


def _big_oracle_for(n: int):
    """The whole queue's trace, cut to an (n)-request batch: the dropped last request is EnvironmentNotFound."""
    tr = [a.copy() for a in _oracle("big", "port")]
    if n == THREE_PASS_N:
        return tr
    if n == 0:
        return [tr[0][: 1 << 20], tr[0][1 << 20:]] + tr[1:]
    assert tr[0]["status"][-1] == STATUS_ENVIRONMENT_NOT_FOUND
    return [tr[0][:n]] + tr[1:]


@pytest.mark.parametrize("packed", [False, True], ids=["plain", "packed"])
@pytest.mark.parametrize("n", [THREE_PASS_N - 1, THREE_PASS_N], ids=["one-launch", "three-pass"])
def test_three_pass_grant_write(make_dispatcher, capfd, n, packed):
    tr, solves = _cuda(make_dispatcher, capfd, None, packed=packed, stream=_big_batch_case(n))
    want = _big_oracle_for(n)
    assert S.traces_equal(tr, want), S.first_mismatch(tr, want)
    (s,) = solves
    assert s["variant"] == 0 and s["final"] == (3 if n == THREE_PASS_N else 1) and s["Nb"] == (1 << 21) * (1 + (n > 1 << 21)), s
    g = tr[0]
    assert (g["status"] == STATUS_GRANTED).sum() > 1_500_000 and (g["status"] == 1).sum() > 100_000


def test_three_pass_queue_as_two_halves(make_dispatcher, capfd):
    """The same queue offered as two consecutive halves of 2^20 requests (each takes the one-launch write)."""
    tr, solves = _cuda(make_dispatcher, capfd, None, stream=_big_batch_case(0))
    want = _big_oracle_for(0)
    assert S.traces_equal(tr, want), S.first_mismatch(tr, want)
    assert [s["final"] for s in solves] == [1, 1]


def test_big_batch_against_reference(make_dispatcher):
    if not REF_LIB.exists():
        pytest.skip("oracle/_ref/libydref.so not built")
    assert S.traces_equal(_oracle("big", "port"), _oracle("big", "ref"))


# ---- fused_max_nb and the merge chunk switch: 262 144 / 262 145 requests -----------------------------------------

def _fused_max_case(coupled: bool, n: int):
    """Solo: cfg2-mod's shape (one digest per servant).  Coupled: 1-3 digests per servant, 20 % of the requestors are
    servants (the merge solver).  The queue's last request is for an unknown digest."""
    def build(d):
        rng = np.random.default_rng(5 + coupled)
        dg = [f"{0x7100 + i:064x}" for i in range(8)]
        svs = []
        for i in range(500):
            envs = [dg[j] for j in rng.choice(8, int(rng.integers(1, 4)), replace=False)] if coupled else [dg[i % 8]]
            svs.append(Servant(f"{S.servant_ip(i)}:8335", None, envs, 8, 128, 0, 256 * GiB, 200 * GiB, 128,
                               PRIORITY_DEDICATED if i % 9 == 0 else PRIORITY_USER))
        env = np.asarray([d.intern_env(x) for x in dg + ["ff" * 32]], dtype=np.uint32)
        outside = np.asarray([d.intern_ip(f"172.18.{i >> 8}.{i & 255}") for i in range(4096)], dtype=np.uint32)
        inside = np.asarray([d.intern_ip(S.servant_ip(i)) for i in range(500)], dtype=np.uint32)
        m = FUSED_MAX_N + 1
        e = env[rng.integers(0, 8, m)]
        e[-1] = env[8]
        ip = outside[rng.integers(0, 4096, m)]
        if coupled:
            ip = np.where(rng.random(m) < 0.2, inside[rng.integers(0, 500, m)], ip)
        return S.Stream("fused-max", _hb(svs) + [("wait", 0.001, S._requests(d, e, ip, 8)[:n]), ("state",)])
    return build


@pytest.mark.parametrize("n", [FUSED_MAX_N, FUSED_MAX_N + 1], ids=["fused", "pipeline"])
@pytest.mark.parametrize("coupled", [False, True], ids=["solo", "merge"])
def test_fused_max_batch(make_dispatcher, capfd, coupled, n):
    tr, solves = _cuda(make_dispatcher, capfd, None, stream=_fused_max_case(coupled, n))
    key = f"fused-max-{'merge' if coupled else 'solo'}"
    for kind in _checkers():
        want = [a.copy() for a in _oracle(key, kind)]
        if n == FUSED_MAX_N:
            assert want[0]["status"][-1] == STATUS_ENVIRONMENT_NOT_FOUND
            want[0] = want[0][:n]
        assert S.traces_equal(tr, want), f"cuda vs {kind}: " + S.first_mismatch(tr, want)
    s = solves[-1]
    if n == FUSED_MAX_N:
        assert s["Nb"] == FUSED_MAX_N and s["variant"] == (1 if coupled else 2) and s["final"] == (1 if coupled else 0), solves
    else:
        assert s["Nb"] == 2 * FUSED_MAX_N and s["variant"] == 0 and s["final"] == 1, solves


# ---- the fused kernel's table bounds ------------------------------------------------------------------------------

def _solo_cluster_case(n_servants: int, extra: int, batches: int, n: int, same: bool):
    """16 digests (16 classes: the initial class bound), servant i holds digest i % 16, capacity 8191 (+ `extra` on
    servant 0); `batches` solo batches of n requests, identical ones if `same`."""
    def build(d):
        rng = np.random.default_rng(n_servants + extra)
        dg = [f"{0x8800 + i:064x}" for i in range(16)]
        svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[i % 16]], 8, 8191 + (extra if i == 0 else 0), 0, 0, 64 * GiB,
                       8191 + (extra if i == 0 else 0)) for i in range(n_servants)]
        env = np.asarray([d.intern_env(x) for x in dg], dtype=np.uint32)
        ips = np.asarray([d.intern_ip(f"172.19.0.{i}") for i in range(200)], dtype=np.uint32)
        ev = _hb(svs)
        reqs = S._requests(d, env[np.arange(n) % 16], ips[rng.integers(0, 200, n)], 8)
        for k in range(batches):
            if not same:
                reqs = S._requests(d, env[rng.integers(0, 16, n)], ips[rng.integers(0, 200, n)], 8)
            ev += [("wait", 0.001 * (k + 1), reqs), ("state",), ("free_frac", k, 0.3)]
        return S.Stream("solo-cluster", ev)
    return build


@pytest.mark.parametrize("extra", [0, 1], ids=["fused", "pipeline"])
def test_fused_slot_tile_bound(make_dispatcher, capfd, monkeypatch, extra):
    """cls_bound x slot tiles <= 32768: static slot bound 2^21 (16 x 2048 tiles) / 2^21 + 1."""
    monkeypatch.setenv("YDSCHED_FUSED_PROF", "1")
    key = f"slot-tiles-{extra}"
    capfd.readouterr()
    d = make_dispatcher("cuda")
    tr = S.Replayer(d, pinned=True, batch_heartbeats=True).run(CASES[key](d))
    d.close()
    err = capfd.readouterr().err
    _check(key, tr)
    solves = _solves(err)
    assert all(s["cls_bound"] == 16 and s["slot_b"] == (1 << 21) << extra for s in solves), solves
    if extra:
        assert all(s["variant"] == 0 and s["final"] == 1 for s in solves) and "fused variant" not in err, solves
    else:
        assert all(s["variant"] >= 2 and s["final"] == 0 for s in solves) and "fused variant" in err, solves


@pytest.mark.parametrize("extra", [0, 1], ids=["speculative", "full"])
def test_speculation_loff_cache_bound(make_dispatcher, capfd, monkeypatch, extra):
    """The speculative solve needs the list offsets in shared memory: 16 x (tiles + 1) + 1 <= 16384 words, i.e. a
    static slot bound of 2^19 (512 tiles) but not 2^19 + 1 (1024 tiles).  Five identical batches."""
    monkeypatch.setenv("YDSCHED_FUSED_PROF", "1")
    key = f"loff-{extra}"
    capfd.readouterr()
    d = make_dispatcher("cuda")
    tr = S.Replayer(d, pinned=True, batch_heartbeats=True).run(CASES[key](d))
    d.close()
    err = capfd.readouterr().err
    _check(key, tr)
    variants = [s["variant"] for s in _solves(err)]
    assert all(v >= 2 for v in variants), variants
    if extra:
        assert 4 not in variants and "(speculative)" not in err, variants
    else:
        assert 4 in variants and "(speculative)" in err, variants


def _class_bound_case(n_digests: int, n: int):
    """n_digests single-digest components (2 servants of capacity 8 each): a 1000-request batch over all of them grows
    the class bound to the first power of two above n_digests + 1, then an n-request batch, then 1000 requests."""
    def build(d):
        rng = np.random.default_rng(n_digests)
        dg = [f"{0x9900 + i:064x}" for i in range(n_digests)]
        svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[i // 2]], 8, 8, 0, 0, 64 * GiB, 8) for i in range(2 * n_digests)]
        env = np.asarray([d.intern_env(x) for x in dg], dtype=np.uint32)
        ips = np.asarray([d.intern_ip(f"172.20.0.{i}") for i in range(200)], dtype=np.uint32)
        ev = _hb(svs)
        for k, m in enumerate((1000, n, 1000)):
            e = env[np.arange(m) % n_digests] if k == 0 else env[rng.integers(0, n_digests, m)]
            ev += [("wait", 0.001 * (k + 1), S._requests(d, e, ips[rng.integers(0, 200, m)], 8)), ("state",),
                   ("free_frac", k, 0.5)]
        return S.Stream("class-bound", ev)
    return build


CLASS_BOUND = {"128-at-256-tiles": (100, 262144, 128, True), "256-at-256-tiles": (200, 262144, 256, False),
               "256-at-128-tiles": (200, 131072, 256, True)}


@pytest.mark.parametrize("case", list(CLASS_BOUND))
def test_fused_request_tile_bound(make_dispatcher, capfd, case):
    """cls_bound x request tiles <= 32768."""
    n_digests, n, bound, fused = CLASS_BOUND[case]
    tr, solves = _cuda(make_dispatcher, capfd, "cls-" + case)
    _check("cls-" + case, tr)
    big = [s for s in solves if s["n"] == n]
    assert len(big) == 1 and big[0]["cls_bound"] == bound, solves
    assert (big[0]["variant"] >= 2) == fused and big[0]["final"] == (0 if fused else 1), big


# ---- kTinyMax: the key-precision walk in batches of 8 and of 9 ------------------------------------------------------

# (and section 3: every solve path on the clusters at the narrow / wide key limit, against port and the exact model)
KEY_PATHS = {  # batch, with_self, dispatcher options
    "tiny": (8, False, {}),
    "nine": (9, False, {}),
    "solo": (K.N_WALK, False, {}),
    "speculative": (1000, False, {}),
    "merge": (K.N_SELF, True, {}),
    "pipeline": (K.N_WALK, False, {"fused": False}),
    "rowscan": (K.N_WALK, False, {"solver": 1}),
    "sequential": (K.N_SELF, True, {"merge_self": False}),
}


@pytest.mark.parametrize("path", list(KEY_PATHS))
@pytest.mark.parametrize("name", list(K.CLUSTERS))
def test_key_precision_on_every_path(make_dispatcher, capfd, name, path):
    batch, with_self, kw = KEY_PATHS[path]
    case = f"keys-{name}-{'self' if with_self else 'walk'}"
    tr, solves = _cuda(make_dispatcher, capfd, case, stream=lambda d: K.key_stream(d, name, batch, with_self),
                       pinned=batch > 9, **kw)  # (thousands of tiny solves: no page-locked buffers per call)
    g = np.concatenate(tr[:-2])
    status, pick, _, _, run = K.model_walk(name, with_self)
    ok = status == STATUS_GRANTED
    assert (g["status"] == status).all() and (g["servant_index"][ok] == pick[ok]).all()
    assert (g["task_id"][ok] == np.arange(int(ok.sum()))).all() and (tr[-2][:, 0] == run).all()
    want = _oracle(case, "port")
    assert (g == want[0]).all() and S.traces_equal(tr[-2:], want[-2:])
    wide = int(K.CLUSTERS[name][1] > 8192)
    assert len(solves) == len(tr) - 2 and all(s["tiny"] == (s["n"] <= 8) for s in solves)  # (kTinyMax = 8)
    if path == "tiny":
        return
    solves = [s for s in solves if s["n"] > 8]  # (the walk in batches of 9 ends with a batch of 7)
    assert solves and all(s["wide"] == wide for s in solves), solves
    v = [s["variant"] for s in solves]
    if path in ("solo",):
        assert v == [2], solves
    elif path == "speculative":
        assert 4 in v, v
    elif path == "merge":
        assert v == [1], solves
    elif path == "pipeline":
        assert v == [0] and solves[0]["solver"] == 2, solves
    elif path == "rowscan":
        assert solves[0]["solver"] == 1 and solves[0]["final"] == 3, solves
    elif path == "sequential":
        assert solves[0]["solver"] == 2, solves


# ---- emask_ok, kMaxClasses, kRowscanMaxComponent, kStreamMaxComponent ----------------------------------------------

def _component_case(kind: str, size: int):
    def build(d):
        rng = np.random.default_rng(size)
        ips = [f"172.21.0.{i}" for i in range(100)]
        if kind == "emask":  # one component holding `size` digests (a ring of servants with two digests each)
            dg = [f"{0xaa00 + i:064x}" for i in range(size)]
            svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[i % size], dg[(i + 1) % size]], 8, 16, 0, 0, 64 * GiB, 16)
                   for i in range(2 * size)]
            digests = lambda m: [dg[j] for j in rng.integers(0, size, m)]
            mv = lambda m: 8
        elif kind == "classes":  # `size` single-digest components: `size` classes
            dg = [f"{0xbb00 + i:064x}" for i in range(size)]
            svs = [Servant(f"{S.servant_ip(i)}:8335", None, [dg[i // 2]], 8, 8, 0, 0, 64 * GiB, 8) for i in range(2 * size)]
            digests = lambda m: [dg[j % size] for j in range(m)]
            mv = lambda m: 8
        else:  # one digest on `size` servants; "stream": two of them behind one IP (the sequential solver)
            dg = ["cc" * 32]
            svs = [Servant(f"{S.servant_ip(i)}:8335", None, dg, 8, 4, int(rng.integers(0, 3)), 0, 64 * GiB, 4,
                           PRIORITY_DEDICATED if i % 9 == 0 else PRIORITY_USER) for i in range(size)]
            if kind == "stream":
                svs[-1] = Servant(f"{S.servant_ip(0)}:9000", None, dg, 8, 4, 0, 0, 64 * GiB, 4)
            ips = ips + [S.servant_ip(i) for i in range(0, size, 97)] + [S.servant_ip(0)] * 20
            digests = lambda m: dg * m
            mv = lambda m: rng.choice([7, 8], m).astype(np.uint32)
        ev = _hb(svs)
        for k, m in enumerate((3000, 1500)):
            ev += [("wait", 0.001 * (k + 1), d.make_requests(m, digests(m), [ips[j] for j in rng.integers(0, len(ips), m)],
                                                              mv(m))), ("state",)]
        return S.Stream(f"{kind}-{size}", ev)
    return build


COMPONENT = {  # case: (kind, size, dispatcher options, check of the debug lines)
    "emask-64": ("emask", 64, {}, lambda s: s["emask"] == 1),
    "emask-65": ("emask", 65, {}, lambda s: s["emask"] == 0),
    "classes-256": ("classes", 256, {}, lambda s: s["solver"] == 2 and s["cls_bound"] == 256),
    "classes-257": ("classes", 257, {}, lambda s: s["solver"] == 1),
    "rowscan-8192": ("rowscan", 8192, {"solver": 1}, lambda s: s["solver"] == 1 and s["max_comp"] == 8192),
    "rowscan-8193": ("rowscan", 8193, {"solver": 1}, lambda s: s["solver"] == 2 and s["max_comp"] == 8193),
    "stream-22000": ("stream", 22000, {}, lambda s: s["solver"] == 2 and s["max_comp"] == 22000),
    "stream-22001": ("stream", 22001, {}, lambda s: s["solver"] == 2 and s["max_comp"] == 22001),
}


@pytest.mark.parametrize("case", list(COMPONENT))
def test_component_limits(make_dispatcher, capfd, case):
    kind, size, kw, ok = COMPONENT[case]
    tr, solves = _cuda(make_dispatcher, capfd, case, **kw)
    _check(case, tr)
    assert len(solves) == 2 and all(ok(s) for s in solves), solves


CASES = {
    **{"slot-" + k: _slot_limit_case(*v) for k, v in SLOT_LIMIT.items()},
    "big": _big_batch_case(THREE_PASS_N),
    "fused-max-solo": _fused_max_case(False, FUSED_MAX_N + 1),
    "fused-max-merge": _fused_max_case(True, FUSED_MAX_N + 1),
    "slot-tiles-0": _solo_cluster_case(256, 0, 3, 2000, False),
    "slot-tiles-1": _solo_cluster_case(256, 1, 3, 2000, False),
    "loff-0": _solo_cluster_case(64, 0, 5, 1000, True),
    "loff-1": _solo_cluster_case(64, 1, 5, 1000, True),
    **{"cls-" + k: _class_bound_case(v[0], v[1]) for k, v in CLASS_BOUND.items()},
    **{f"keys-{n}-{m}": (lambda n, m: lambda d: K.key_stream(d, n, K.N_WALK, m == "self"))(n, m)
       for n in K.CLUSTERS for m in ("walk", "self")},
    **{k: _component_case(v[0], v[1]) for k, v in COMPONENT.items()},
}
