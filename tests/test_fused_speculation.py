"""The speculative solo solve (fused.cuh): a batch whose class set is the one of the previous solo solves runs against
the class table those solves kept, with one grid barrier.  A stream that takes the speculative path, misses it in every
way a batch can (new digest, new min_version, a requestor that is a servant of its component), changes the topology and
the class bound, frees and ticks in between -- replayed through the CUDA backend and compared with the CPU checker."""
import numpy as np
import pytest

from yadcc_b200 import STATUS_GRANTED, Servant
from yadcc_b200 import streams as S

pytestmark = pytest.mark.gpu

N_DIGESTS = 24  # one component per digest: every batch below is data-parallel
N_SERVANTS = 192


def _servant(i: int, digest: str) -> Servant:
    return Servant(f"{S.servant_ip(i)}:8335", None, [digest], 10, 64, 0, 256 << 30, 200 << 30, 24)


def _speculation_stream(d, seed=11):
    rng = np.random.default_rng(seed)
    dgs = [f"{0x5eed0000 + i:064x}" for i in range(N_DIGESTS)]
    ev = [("hb", 0.0, _servant(i, dgs[i % N_DIGESTS]), 100.0) for i in range(N_SERVANTS)]
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    outside = np.asarray([d.intern_ip(f"172.16.1.{i}") for i in range(200)], dtype=np.uint32)
    inside = np.asarray([d.intern_ip(S.servant_ip(i)) for i in range(N_SERVANTS)], dtype=np.uint32)
    unknown = d.intern_env(f"{0xdead:064x}")  # a digest nobody holds: EnvironmentNotFound, not a miss
    now = 0.001

    def batch(digests, min_version=8, self_frac=0.0, extra_mv=None):
        nonlocal now
        n = 1000  # (one batch size class: the class table sits behind res[], whose size follows it)
        e = env[rng.choice(digests, n)]
        e[rng.random(n) < 0.01] = unknown
        mv = np.full(n, min_version, np.uint32)
        if extra_mv is not None:  # (digest, min_version) of every request for that digest
            mv[e == env[extra_mv[0]]] = extra_mv[1]
        ips = outside[rng.integers(0, len(outside), n)]
        if self_frac:
            ips = np.where(rng.random(n) < self_frac, inside[rng.integers(0, N_SERVANTS, n)], ips)
        ev.append(("wait", now, S._requests(d, e, ips, mv, expires_in_s=float(rng.choice([0.02, 15.0])),
                                            prefetch=rng.random(n) < 0.2)))
        ev.append(("state",))
        ev.append(("free_frac", int(rng.integers(1 << 30)), 0.5))
        ev.append(("tick", now + 0.005))
        now += 0.01

    first = list(range(8))
    for _ in range(4):             # same class set: the third and fourth solves speculate
        batch(first)
    batch(first + [8])             # a new digest: miss, replay
    for _ in range(3):
        batch(first + [8])         # two agreeing solves, then speculation again
    batch(first + [8], extra_mv=(2, 9))  # a new min_version for a known digest: miss
    for _ in range(3):
        batch(first + [8], extra_mv=(2, 9))
    batch(first + [8], extra_mv=(2, 9), self_frac=0.1)  # requests from servants of their components: miss
    for _ in range(3):
        batch(first + [8], extra_mv=(2, 9))
    ev.append(("hb", now, _servant(N_SERVANTS, dgs[0]), 100.0))  # a new servant: a new topology, no speculation
    for _ in range(3):
        batch(first + [8], extra_mv=(2, 9))
    batch(list(range(N_DIGESTS)))  # more classes than the class bound: it grows, the kept table is dropped
    for _ in range(4):
        batch(list(range(N_DIGESTS)))
    return S.Stream("speculation", ev)


@pytest.mark.parametrize("packed", [True, False], ids=["packed", "plain"])
@pytest.mark.parametrize("graphs", [True, False], ids=["graph", "eager"])
def test_speculative_solo_solve_equals_oracle(make_dispatcher, monkeypatch, capfd, packed, graphs):
    monkeypatch.setenv("YDSCHED_FUSED_PROF", "1")
    traces, launches = {}, []
    for kind in ("cuda", "port"):
        d = make_dispatcher(kind, graphs=graphs) if kind == "cuda" else make_dispatcher(kind)
        on_solve = (lambda dd, reqs, g: launches.append(dd.last_solve_stats()["kernel_launches"])) if kind == "cuda" else None
        traces[kind] = S.Replayer(d, pinned=(kind == "cuda"), packed=(packed and kind == "cuda"),
                                  on_solve=on_solve).run(_speculation_stream(d))
        d.close()
    assert S.traces_equal(traces["cuda"], traces["port"]), S.first_mismatch(traces["cuda"], traces["port"])
    lines = [x for x in capfd.readouterr().err.splitlines() if "fused variant 4 (speculative)" in x]
    hits = [x for x in lines if not x.endswith("missed")]
    misses = [x for x in lines if x.endswith("missed")]
    assert hits, lines              # the steady stretches of the stream were decided speculatively ...
    assert misses, lines            # ... and a changed class set was caught and replayed
    assert 2 in launches, launches  # (a miss and its replay: two launches in one call)


def test_changing_class_sets_never_speculate(make_dispatcher, monkeypatch, capfd):
    """Batches whose class set differs from the previous one's: no solve keeps its class table, so none speculates
    (and none pays for a miss)."""
    monkeypatch.setenv("YDSCHED_FUSED_PROF", "1")
    d = make_dispatcher("cuda")
    dgs = [f"{0x5eed0000 + i:064x}" for i in range(N_DIGESTS)]
    for i in range(N_SERVANTS):
        d.keep_servant_alive(_servant(i, dgs[i % N_DIGESTS]), 100.0, now=0.0)
    for k in range(8):
        reqs = d.make_requests(500, [dgs[(k + j) % 8] for j in range(500)], "172.16.0.9", 8 + k % 2)
        g = d.wait_for_starting_new_tasks(reqs, 0.001 * (k + 1))
        if k:  # (the first solve also builds the slot order)
            assert d.last_solve_stats()["kernel_launches"] == 1
        d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED].copy())
    err = capfd.readouterr().err
    assert "fused variant 2" in err and "speculative" not in err
