"""The test-only NCCL stand-in (tests/fake_nccl) without a GPU: it is the libnccl.so.2 a process gets once it is
preloaded, and its rendezvous gathers rank-major, sums in place mod 2^32, takes zero-length calls and ends the process
with a report when the ranks' calls disagree."""
import ctypes as C
import os
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "tests" / "fake_nccl" / "libnccl.so.2"


def run_py(code: str, timeout=60):
    return subprocess.run([sys.executable, "-c", textwrap.dedent(code)], capture_output=True, text=True, timeout=timeout,
                          cwd=ROOT, env=dict(os.environ, FAKE_NCCL=str(LIB)))


@pytest.fixture(scope="module", autouse=True)
def built():
    assert LIB.exists(), f"{LIB} missing: run build() or `make fake_nccl`"


def test_preloaded_stand_in_is_the_libnccl_a_dlopen_finds():
    p = run_py("""
        import ctypes, os
        ctypes.CDLL(os.environ["FAKE_NCCL"], mode=ctypes.RTLD_GLOBAL)
        lib = ctypes.CDLL("libnccl.so.2")
        print(hasattr(lib, "yd_fake_nccl_stats"), hasattr(lib, "ncclAllReduce"))
    """)
    assert p.returncode == 0 and p.stdout.split() == ["True", "True"], p.stdout + p.stderr


RANKS_CODE = """
    import ctypes as C, os, sys, threading
    import numpy as np
    lib = C.CDLL(os.environ["FAKE_NCCL"], mode=C.RTLD_GLOBAL)
    lib.yd_fake_nccl_host_buffers(1)
    W = {world}
    class UniqueId(C.Structure):  # passed by value to ncclCommInitRank
        _fields_ = [("internal", C.c_uint8 * 128)]
    uid = UniqueId()
    lib.ncclCommInitRank.argtypes = [C.c_void_p, C.c_int, UniqueId, C.c_int]
    assert lib.ncclGetUniqueId(C.byref(uid)) == 0
    comms = [C.c_void_p() for _ in range(W)]
    def init(r):
        assert lib.ncclCommInitRank(C.byref(comms[r]), W, uid, r) == 0
    ts = [threading.Thread(target=init, args=(r,)) for r in range(W)]
    [t.start() for t in ts]; [t.join() for t in ts]
    lib.ncclAllGather.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    lib.ncclAllReduce.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    def on_ranks(f):
        out = [None] * W
        def run(r):
            out[r] = f(r)
        ts = [threading.Thread(target=run, args=(r,)) for r in range(W)]
        [t.start() for t in ts]; [t.join() for t in ts]
        return out
"""


def test_rendezvous_on_host_buffers():
    p = run_py(RANKS_CODE.format(world=3) + """
    rng = np.random.default_rng(1)
    send = [rng.integers(0, 2**32, 5, dtype=np.uint64).astype(np.uint32) for _ in range(W)]
    recv = [np.zeros(5 * W, dtype=np.uint32) for _ in range(W)]
    rc = on_ranks(lambda r: lib.ncclAllGather(send[r].ctypes.data, recv[r].ctypes.data, 5, 3, comms[r], None))
    assert rc == [0] * W
    for r in range(W):
        assert (recv[r] == np.concatenate(send)).all()  # rank-major
    buf = [np.array([0xFFFFFFFF, r, 7], dtype=np.uint32) for r in range(W)]
    rc = on_ranks(lambda r: lib.ncclAllReduce(buf[r].ctypes.data, buf[r].ctypes.data, 3, 3, 0, comms[r], None))
    assert rc == [0] * W
    for r in range(W):
        assert buf[r].tolist() == [(0xFFFFFFFF * W) % 2**32, sum(range(W)), 7 * W]  # in place, mod 2^32
    rc = on_ranks(lambda r: lib.ncclAllReduce(None, None, 0, 3, 0, comms[r], None))
    assert rc == [0] * W
    st = (C.c_ulonglong * 4)()
    lib.yd_fake_nccl_stats(1, st)
    assert list(st) == [3, 1, 2, 5 * 4 * W + 3 * 4], list(st)
    assert on_ranks(lambda r: lib.ncclCommDestroy(comms[r])) == [0] * W
    print("OK")
    """)
    assert p.returncode == 0 and p.stdout.strip() == "OK", p.stdout + p.stderr


def test_mismatched_calls_end_the_process_with_a_report():
    p = run_py(RANKS_CODE.format(world=2) + """
    a = [np.zeros(8, dtype=np.uint32) for _ in range(W)]
    on_ranks(lambda r: lib.ncclAllReduce(a[r].ctypes.data, a[r].ctypes.data, 4 + r, 3, 0, comms[r], None))
    print("not reached")
    """)
    assert p.returncode == 86 and "not reached" not in p.stdout, p.stdout + p.stderr
    assert "ranks disagree" in p.stderr and "rank 0: call #1 AllReduce count 4" in p.stderr \
        and "rank 1: call #1 AllReduce count 5" in p.stderr, p.stderr
