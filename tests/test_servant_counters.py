"""The speculative solo solve's servant counters (fused.cuh: fused_servant_counters): instead of two atomics per grant,
each servant's grants are counted once, from the sorted position of the last member its class grants.  Streams that
reach the speculative solve (variant 4) with that boundary in every place it can fall, replayed through the CUDA backend
in plain, packed and staged calls and compared with the CPU restatement, servant bookkeeping (running_tasks,
ever_assigned_tasks) included after every solve; the solve lines show that the solves they target ran speculatively.

  fewer       fewer requests than slots per class: the boundary falls inside a servant's run of slots
  more        more requests than slots: timeouts, every member taken
  versions    a class whose servants are all below its min_version (cls_nelig 0: k_s = 0) and one with some below
  busy        only part of each batch freed: servants enter the solve partly busy
  mixed       mixed nproc / max_tasks, servants with equal facts (equal codes, broken by the original slot index)
  dedicated   dedicated servants (the capacity tier changes along the row) and load > 0
  classes80   more than 64 kept classes
  two-tiles   140 k requests: more request tiles than blocks, every block counts servants after its tiles
  cfg4        bench.py's filtered call sequence (its compacted queue is decided speculatively)"""
import numpy as np
import pytest

from solve_lines import solves
from yadcc_b200 import Servant
from yadcc_b200 import _abi
from yadcc_b200 import streams as S

pytestmark = pytest.mark.gpu

GIB = 1 << 30
SOLVES = 5  # per stream: two solo solves that agree on the class set, then speculative ones


def _servant(i, digest, version=9, nproc=16, load=0, max_tasks=16, priority=_abi.PRIORITY_USER):
    return Servant(f"{S.servant_ip(i)}:8335", None, [digest], version, nproc, load, 64 * GIB, 40 * GIB, max_tasks,
                   priority)


def _case(name, rng):
    """(servants as (digest index, Servant kwargs), number of digests, requests per batch, min_version per digest,
    fraction of the grants freed between batches)."""
    K, n, free, mv = 8, 600, 1.0, None
    kw = lambda i: {}  # noqa: E731
    n_sv = 64
    if name == "more":
        n = 3000
    elif name == "versions":
        mv = {k: 8 for k in range(K)}
        kw = lambda i: {"version": 5 if i % K == 7 else [7, 8, 9][i % 3] if i % K == 6 else 9}  # noqa: E731
    elif name == "busy":
        n, free = 500, 0.4
    elif name == "mixed":
        n_sv, n = 96, 900
        facts = [(int(rng.integers(1, 25)), int(rng.integers(1, 25))) for _ in range(6)]  # a few shapes, many twins
        kw = lambda i: dict(zip(("nproc", "max_tasks"), facts[i % 6]))  # noqa: E731
    elif name == "dedicated":
        n_sv, n = 96, 900

        def kw(i):
            if i % 3 == 0:
                nproc = 33 if i % 2 else 32
                return {"nproc": nproc, "max_tasks": nproc * 95 // 100, "load": nproc // 2 + i % 3 - 1,
                        "priority": _abi.PRIORITY_DEDICATED}
            return {"nproc": 16, "max_tasks": 12, "load": i % 5}
    elif name == "classes80":
        K, n_sv, n = 80, 240, 2000
    elif name == "two-tiles":
        n_sv, n = 600, 140_000
        kw = lambda i: {"nproc": 96, "max_tasks": 96}  # noqa: E731
    mv = mv or {k: 8 for k in range(K)}
    return [(i % K, kw(i)) for i in range(n_sv)], K, n, mv, free


def _stream(d, name, seed=5):
    rng = np.random.default_rng(seed)
    servants, K, n, mv, free = _case(name, rng)
    dgs = [f"{0xc0de0000 + k:064x}" for k in range(K)]
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    clients = np.asarray([d.intern_ip(f"172.31.0.{k}") for k in range(100)], dtype=np.uint32)
    ev = [("hb", 0.0, _servant(i, dgs[k], **f), 1e6) for i, (k, f) in enumerate(servants)]
    # the id staging of FreeTask / KeepTaskAlive at its largest size first: a device buffer that grows drops the kept
    # class table
    bogus = np.arange(1 << 40, (1 << 40) + (1 << 17), dtype=np.uint64)
    ev += [("free", bogus), ("keepalive", 0.0, bogus, 1.0)]
    weights = rng.random(K) + 0.2
    now = 0.001
    for _ in range(SOLVES):
        k = rng.choice(K, n, p=weights / weights.sum())
        k[rng.permutation(n)[:K]] = np.arange(K)  # every class in every batch: one class set
        reqs = S._requests(d, env[k], clients[rng.integers(0, len(clients), n)],
                           np.asarray([mv[int(x)] for x in range(K)], dtype=np.uint32)[k], expires_in_s=15.0,
                           prefetch=rng.random(n) < 0.2)
        ev += [("wait", now, reqs), ("state",), ("free_frac", int(rng.integers(1 << 30)), free), ("tick", now + 0.005)]
        now += 0.01
    return S.Stream(f"counters-{name}", ev)


CASES = ["fewer", "more", "versions", "busy", "mixed", "dedicated", "classes80", "two-tiles"]
MODES = ["plain", "packed", "staged"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_servant_counters_equal_restatement(make_dispatcher, capfd, monkeypatch, name, mode):
    if name == "two-tiles" and mode != "staged":
        pytest.skip("one call mode is enough for the 140 k-request batches (the restatement decides them slowly)")
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    calls = []
    d = make_dispatcher("cuda")
    capfd.readouterr()
    got = S.Replayer(d, pinned=True, packed=mode == "packed", staged=mode == "staged",
                     on_solve=lambda dd, reqs, g: calls.append(solves(capfd.readouterr().err))).run(_stream(d, name))
    d.close()
    monkeypatch.delenv("YDSCHED_DEBUG")
    p = make_dispatcher("port")
    want = S.Replayer(p).run(_stream(p, name))
    p.close()
    assert S.traces_equal(got, want), S.first_mismatch(got, want)
    assert len(calls) == SOLVES and all(len(x) == 1 for x in calls), calls
    paths = [(x[0]["variant"], x[0]["spec"]) for x in calls]
    assert all(p == (4, 1) for p in paths[2:]), paths  # the solves after two agreeing ones are speculative hits


def test_cfg4_filtered_solve_counters(cuda_lib, port_lib, capfd, monkeypatch):
    """bench.py's cfg4 call sequence: the filtered call's compacted queue is decided speculatively, and the servant
    state after every step equals the restatement's."""
    from test_staged_solves import _bench_sequence

    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    rec, states, lines = _bench_sequence(cuda_lib, "cfg4", capfd)
    monkeypatch.delenv("YDSCHED_DEBUG")
    want, want_states, _ = _bench_sequence(port_lib, "cfg4")
    for (what, step, g), (_, _, h) in zip(rec, want):
        assert g.shape == h.shape and (g == h).all(), (what, step, S.first_mismatch([g], [h]))
    for step, (a, b) in enumerate(zip(states, want_states)):
        assert (a == b).all(), ("servant_state after step", step)
    assert any(x and x[0]["variant"] == 4 and x[0]["spec"] == 1 for x in lines), lines
