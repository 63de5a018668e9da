"""Runs of Heartbeat, KeepTaskAlive and FreeTask frames served as one batch each (yd_wire_handle_frames over
yd_service_heartbeats / yd_service_keep_tasks_alive / yd_service_free_tasks), checked frame by frame and state by state
against yd_wire_call one frame at a time (tests/service_runs_cases.py).  On the CPU: the port (its state build, which
also exports the whole decision state) and the reference build.  On the GPU: the CUDA library's frames against the
port's calls, and against its own calls."""
import subprocess

import numpy as np
import pytest

pytest.importorskip("google.protobuf")

import service_runs_cases as R  # noqa: E402
from conftest import CUDA_LIB, REF_LIB, ROOT  # noqa: E402
from yadcc_b200 import TaskDispatcher  # noqa: E402

PORT_STATE_LIB = ROOT / "checkers" / "libydport_state.so"
SEEDS = [1, 2, 3, 4, 5, 6]


@pytest.fixture
def make_lib(request):
    made = []

    def lib_of(kind):
        if kind == "port":
            if not PORT_STATE_LIB.exists():
                subprocess.check_call(["make", "-C", str(ROOT), "checkers/libydport_state.so"])
            return str(PORT_STATE_LIB)
        if kind == "ref":
            if not REF_LIB.exists():
                pytest.skip("oracle/_ref/libydref.so not built")
            return str(REF_LIB)
        assert CUDA_LIB.exists(), "yadcc_b200/libydsched.so missing: run build()"
        return str(CUDA_LIB)

    def factory(kind):
        def make():
            d = TaskDispatcher(lib_of(kind))
            made.append(d)
            return d
        return make

    yield factory
    for d in made:
        d.close()


def _random(make_lib, a, b, seed, n_windows=40):
    t = R.Twins(make_lib(a), make_lib(b), seed=seed)
    try:
        frames = R.run_random(t, seed, n_windows)
    finally:
        t.close()
    assert frames > 200


def _targeted(make_lib, a, b, name):
    t = R.Twins(make_lib(a), make_lib(b))
    try:
        R.TARGETED[name](t)
    finally:
        t.close()


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_runs_header_is_exported_by_the_product_and_the_port_builds():
    """include/ydruns.h is declared one-to-one in _abi.RUNS_PROTOTYPES and is not part of what ydsched.h, ydservice.h or
    ydwire.h require of every library (reference builds from earlier trees lack it).  The CUDA library (required by
    load_library) and every port build export it."""
    import ctypes as C

    from test_abi import header_symbols
    from yadcc_b200 import _abi

    names = header_symbols("ydruns.h")
    assert names == sorted(name for name, _, _ in _abi.RUNS_PROTOTYPES)
    assert not set(names) & set(header_symbols() + header_symbols("ydservice.h") + header_symbols("ydwire.h"))
    for lib in (CUDA_LIB, ROOT / "oracle" / "libydoracle.so", PORT_STATE_LIB, ROOT / "checkers" / "libydport_keys.so"):
        h = C.CDLL(str(lib))
        assert all(hasattr(h, name) for name in names), lib


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("kind", ["port", "ref"])
def test_random_streams(make_lib, kind, seed):
    _random(make_lib, kind, kind, seed)


@pytest.mark.parametrize("name", sorted(R.TARGETED))
@pytest.mark.parametrize("kind", ["port", "ref"])
def test_targeted(make_lib, kind, name):
    _targeted(make_lib, kind, kind, name)


@pytest.mark.parametrize("kind", ["port", "ref"])
def test_keep_tasks_alive_is_the_loop(make_lib, kind):
    """Each checker's yd_keep_tasks_alive against its own loop of yd_keep_task_alive.  A reference build from a tree
    that predates yd_keep_tasks_alive (ydruns.h is optional for the checkers) still gives the loop: the port's call is
    compared against the reference's own single calls."""
    make = make_lib(kind)
    probe = make()
    a = make if hasattr(probe._lib, "yd_keep_tasks_alive") else make_lib("port")
    for seed in range(4):
        R.keep_tasks_alive_case(make, seed, make_a=a)


def test_batched_runs_match_the_reference_build(make_lib):
    """The port's batched frames against the reference build's single calls."""
    _random(make_lib, "port", "ref", 11)


def test_service_calls_match_single_handlers(make_lib):
    """The three service calls at the Python level: each answer equals the single handler's on a twin."""
    from yadcc_b200.service import HeartbeatRequest

    t = R.Twins(make_lib("port"), make_lib("port"))
    try:
        R._cluster(t, 3)
        ids = R._grant(t, 0.5, 4)
        a, b = t.a, t.b
        reqs = [HeartbeatRequest(token=tok, location=f"10.7.0.{k}:8335", remote_ip=f"10.7.0.{k}", next_heartbeat_in_ms=5000,
                                 version=3, num_processors=8, capacity=4, servant_priority=2,
                                 total_memory_in_bytes=1 << 36, memory_available_in_bytes=1 << 35, env_digests=[R.ENVS[0]],
                                 running_tasks=[])
                for k, tok in [(0, "s1"), (1, "bad"), (2, "u1"), (5, "s1")]]
        assert a.heartbeats(reqs, now=1.0) == [b.heartbeat(r, now=1.0) for r in reqs]
        kreq = [("u1", ids + [ids[0], 10**9], 2000), ("bad", ids, 1000), ("u2", ids[:1], 30001), ("u1", [], 1000)]
        got = a.keep_tasks_alive(kreq, now=1.5)
        want = [b.keep_task_alive(*r, now=1.5) for r in kreq]
        assert [(s, list(o) if s == 0 else None) for s, o in got] == [(s, list(o) if s == 0 else None) for s, o in want]
        freq = [("u1", ids[:2] + ids[:1]), ("bad", ids[2:]), ("u1", [10**9])]
        assert a.free_tasks(freq) == [b.free_task(*r) for r in freq]
        t.compare(1.5)
    finally:
        t.close()


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("against", ["port", "cuda"])
def test_gpu_random_streams(make_lib, against, seed):
    _random(make_lib, "cuda", against, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(R.TARGETED))
@pytest.mark.parametrize("against", ["port", "cuda"])
def test_gpu_targeted(make_lib, against, name):
    _targeted(make_lib, "cuda", against, name)


@pytest.mark.gpu
def test_gpu_keep_tasks_alive_is_the_loop(make_lib):
    for seed in range(4):
        R.keep_tasks_alive_case(make_lib("cuda"), seed)


@pytest.mark.gpu
def test_gpu_keep_tasks_alive_against_the_port(make_lib):
    """The CUDA call with a length per id against the port's loop, on many repeated ids: the last length wins."""
    rng = np.random.default_rng(7)
    t = R.Twins(make_lib("cuda"), make_lib("port"))
    try:
        R._cluster(t, 6, ms=30000)
        ids = R._grant(t, 0.5, 24, ka_ms=30000)
        for step in range(6):
            now = 1.0 + step
            sel = [ids[int(i)] for i in rng.integers(0, len(ids), size=3000)]
            lens = [float(rng.choice([0.0, 0.25, 1.0, 2.0, 30.0])) for _ in sel]
            got = t.a.dispatcher.keep_tasks_alive(sel, lens, now=now)
            want = t.b.dispatcher.keep_tasks_alive(sel, lens, now=now)
            assert (got == want).all()
            t.compare(now)
            for dt in (0.25, 1.0, 1.0 + 1e-9):
                t.tick(now + dt)
    finally:
        t.close()
