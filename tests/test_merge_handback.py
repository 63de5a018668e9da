"""Both sides of every rule by which the merge solver hands a component back to the sequential solver
(solve_merge.cuh: pending runs, the skip limit, the last-resort check; classes.cuh: classes per component), on the
cases of merge_cases.py.  Every case is compared with the CPU restatement (and the reference where it is built) --
statuses, task ids, servant indices and servant_state() -- through the plain and the packed call, and again with
merge_self=False, where the sequential solver decides the component alone.  Each case reads the YDSCHED_DEBUG solve
line and asserts which side it ran: merge_back (the OR of the kBack* reasons over the handed-back components),
merge_back_n (how many) and merge_chunks (the merge solver ran).  The range-sharded record window is tested through
tests/shard_merge_check.py.
"""
import functools
import json
import os
import subprocess
import sys

import pytest

import merge_cases as M
from conftest import REF_LIB, ROOT, _ensure_port
from solve_lines import solves as _solves
from yadcc_b200 import TaskDispatcher
from yadcc_b200 import streams as S

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _oracle(name: str, lib: str):
    d = TaskDispatcher(lib)
    try:
        return S.Replayer(d, batch_heartbeats=True).run(M.stream(d, M.CASES[name]))
    finally:
        d.close()


# The sequential solver cannot take the skip-limit cases in reasonable time: a million requests from one servant's IP
# leave that servant's free slot at the front of the class's slot list, and every exact walk starts there and steps over
# every slot taken since (quadratic in the run).  Those cases run the merge solver's side only; the model test shows
# which side of the limit each one is on.
PARAMS = [(n, m) for n in M.CASES for m in ("plain", "packed", "sequential")
          if not (n.startswith("skip-") and (M.CASES[n].back or m == "sequential"))]


@pytest.mark.parametrize("name,mode", PARAMS)
def test_merge_handback(make_dispatcher, capfd, monkeypatch, name, mode):
    c = M.CASES[name]
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    if c.chunk:
        monkeypatch.setenv("YDSCHED_MERGE_CHUNK", str(c.chunk))
    capfd.readouterr()
    # (tiny=False: the batches of the check cases are below the tiny path's limit)
    d = make_dispatcher("cuda", tiny=False, merge_self=mode != "sequential")
    tr = S.Replayer(d, packed=mode == "packed", batch_heartbeats=True).run(M.stream(d, c))
    d.close()
    for lib in [str(_ensure_port())] + ([str(REF_LIB)] if REF_LIB.exists() else []):
        want = _oracle(name, lib)
        assert S.traces_equal(tr, want), f"cuda vs {lib}: " + S.first_mismatch(tr, want)
    (s,) = _solves(capfd.readouterr().err)
    assert s["n"] == len(c.reqs) and s["solver"] == 2, s
    if mode == "sequential":
        assert s["merge_chunks"] == 0 and s["merge_back"] == 0 and s["merge_back_n"] == 0, s
        return
    assert s["merge_back"] == c.back and s["merge_back_n"] == int(c.back != 0), s
    assert (s["merge_chunks"] > 0) == c.merge, s
    if c.chunk == 32:
        assert s["merge_rounds"] >= 2, s


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_record_window(world):
    """The merge solver reads a class's records up to its slot-list length + kRqMargin on a range-sharded group
    (tests/shard_merge_check.py: W ranks over the test-only NCCL stand-in, checked against one checker fed the whole
    queue).  One record short of that the group decides the batch; at it every rank falls back to the whole queue (an
    odd number of all-gathers, the ranges' one included) and names the window as the reason.  A saturated class on a
    large component reads nowhere near the window, so the group decides it too."""
    for p in (ROOT / "tests" / "fake_nccl" / "libnccl.so.2", ROOT / "oracle" / "libydoracle.so"):
        assert p.exists(), f"{p} missing: run build()"
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "shard_merge_check.py"), "--world", str(world)],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, YDSCHED_DEBUG="1"))
    lines = [json.loads(x) for x in p.stdout.splitlines() if x.startswith("{")]
    msg = p.stdout[-4000:] + p.stderr[-3000:]
    assert p.returncode == 0 and lines and lines[-1]["shard_parity"] is True, msg
    assert lines[-1]["fake_nccl_collectives"] > 0 and not lines[-1]["torch_loaded"], msg
    got = {c["case"]: c for c in lines[:-1]}
    assert list(got) == list(M.SHARDED) and all(c["ok"] and c["solves"] == 1 for c in got.values()), msg
    assert {k: c["handbacks"] for k, c in got.items()} == {"margin-1023": 0, "margin-1024": 1, "saturated": 0}, msg
    # every rank names the rule: a record that was not gathered (kBackWindow), on the one component
    n = len(M.SHARDED["margin-1024"].reqs)
    rows = [x.split() for x in p.stderr.splitlines() if x.startswith("ydsched: shard rank ")]
    back = sorted((int(t[3]), int(t[7]), int(t[9]), int(t[11]), int(t[13])) for t in rows)  # rank, n, flag, reasons, comps
    assert back == [(r, n, 4, 4, 1) for r in range(world)], (back, msg)
