"""The one-launch solo solve's state from one call to the next (fused.cuh, ydsched.cu WaitImpl): the kept slot order,
the kept class table of the speculative solve, the clean scratch, the solo hint, the servant facts and topology on the
device, and the lease ring.  Each seed of `streams.solo_stream` runs steady stretches of data-parallel batches, each
ended by one perturbation from `streams.SOLO_MENU`, through the CUDA backend and through the CPU restatement (and the
reference on every third seed, where it is built), and asserts from the YDSCHED_DEBUG lines that the batch after each
perturbation took the path the menu names -- a case that drifts onto another path fails instead of passing there.
A third of the seeds hand out more than 2^17 task ids (the lease ring's live window crosses the ring's end); every
sixth grows the ring while its live window straddles the ring's end."""
import collections
import functools

import pytest

from conftest import REF_LIB
from solve_lines import solves
from yadcc_b200 import streams as S

pytestmark = pytest.mark.gpu

SEEDS = range(24)
STRIDED = (5, 16)  # id_stride 4, id_offset 3 on both backends
COUNTS: collections.Counter = collections.Counter()


def _interface(seed: int) -> dict:
    """graph / eager x plain / packed x page-locked (zero-copy) / pageable: each combination on three seeds."""
    return {"graphs": seed % 2 == 0, "packed": seed // 2 % 2 == 1, "pinned": seed // 4 % 2 == 0}


def _ids(seed: int) -> dict:
    return {"id_stride": 4, "id_offset": 3} if seed in STRIDED else {}


@functools.lru_cache(maxsize=4)
def _oracle(seed: int, kind: str):
    from conftest import _ensure_port
    from yadcc_b200 import TaskDispatcher

    d = TaskDispatcher(str(_ensure_port()) if kind == "port" else str(REF_LIB), **_ids(seed))
    try:
        return S.Replayer(d).run(S.solo_stream(d, seed))
    finally:
        d.close()


def _check_path(lines: list, launches: list, at: int, item: str, want: str) -> None:
    s = lines[at]
    ctx = f"{item} -> batch {at}: {s}"
    assert s["tiny"] == 0, ctx
    if s["ring_cap"] != lines[at - 1]["ring_cap"]:
        # the lease ring grew in this very solve: its buffers moved, and with them every signature of the kept state
        assert s["spec"] == 0 and s["variant"] in (1, 2), ctx
        return
    if want in ("hit", "rebuild"):
        assert s["spec"] == 1 and s["variant"] == 4 and s["final"] == 0, ctx
        # (a rebuild of the kept slot order is a launch of its own before the kernel)
        assert (launches[at] == 1) == (want == "hit"), f"{ctx}, {launches[at]} launches"
    elif want == "replay":
        assert s["spec"] == 2 and s["variant"] == 3 and s["final"] == 0, ctx
    elif want == "standdown":
        assert s["spec"] == 2 and s["variant"] == 1, ctx
        assert lines[at + 1]["variant"] == 1 and lines[at + 2]["variant"] in (2, 3), (ctx, lines[at + 1: at + 3])
    elif want == "fresh":
        assert s["spec"] == 0 and s["variant"] == 2, ctx
    elif item == "size-class":
        assert s["spec"] == 0 and s["variant"] == 2 and s["Nb"] != lines[at - 1]["Nb"], ctx
    else:  # class-bound: the speculative solve misses, the bound grows, the batch (two classes on a digest) stands down
        assert s["spec"] == 2 and s["cls_bound"] > lines[at - 1]["cls_bound"], ctx


@pytest.mark.parametrize("seed", SEEDS)
def test_solo_state_across_calls(make_dispatcher, capfd, monkeypatch, seed):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    io = _interface(seed)
    capfd.readouterr()
    d = make_dispatcher("cuda", graphs=io["graphs"], **_ids(seed))
    stream = S.solo_stream(d, seed)
    calls = []  # (kernel launches, the next task id's ordinal) after every solve
    stride, offset = _ids(seed).get("id_stride", 1), _ids(seed).get("id_offset", 0)
    on_solve = lambda dd, r, g: calls.append((dd.last_solve_stats()["kernel_launches"],  # noqa: E731
                                              (dd.next_task_id() - offset) // stride))
    tr = S.Replayer(d, pinned=io["pinned"], packed=io["packed"], on_solve=on_solve).run(stream)
    d.close()
    lines = solves(capfd.readouterr().err)
    for kind in ("port", "ref") if seed % 3 == 0 and REF_LIB.exists() and seed not in STRIDED else ("port",):
        want = _oracle(seed, kind)
        assert S.traces_equal(tr, want), f"cuda vs {kind}: " + S.first_mismatch(tr, want)

    assert len(lines) == len(calls) == stream.meta["waits"]
    launches = [c[0] for c in calls]
    for at, item, want in stream.meta["checks"]:
        _check_path(lines, launches, at, item, want)
    assert {item for _, item, _ in stream.meta["checks"]} == set(S.SOLO_MENU)

    nexts = [c[1] for c in calls]
    wrapped = [i for i, s in enumerate(lines) if nexts[i] > s["ring_cap"] and s["ring_lo"] > 0]
    grown = [i for i in range(1, len(lines)) if lines[i]["ring_cap"] > lines[i - 1]["ring_cap"]]
    # the window [ring_lo, next) the growing solve found, in the old ring: its two ends in different laps
    straddled = [i for i in grown
                 if lines[i]["ring_lo"] // lines[i - 1]["ring_cap"] != (nexts[i - 1] - 1) // lines[i - 1]["ring_cap"]]
    if stream.meta["wrap"]:
        assert nexts[-1] > 1 << 17 and wrapped, (nexts[-1], lines[-1])
    if stream.meta["grow"]:
        assert straddled, [(lines[i - 1]["ring_cap"], lines[i]["ring_lo"], nexts[i - 1]) for i in grown]

    COUNTS["seeds"] += 1
    COUNTS["solves"] += len(lines)
    COUNTS.update(f"variant {s['variant']}" for s in lines if not s["tiny"])
    COUNTS["tiny"] += sum(s["tiny"] for s in lines)
    COUNTS["speculative hits"] += sum(s["spec"] == 1 for s in lines)
    COUNTS["speculative misses"] += sum(s["spec"] == 2 for s in lines)
    COUNTS["flag-4 stand-downs after a miss"] += sum(s["spec"] == 2 and s.get("variant") == 1 for s in lines)
    COUNTS["wrap seeds past 2^17 ids"] += bool(stream.meta["wrap"] and wrapped)
    COUNTS["ring growths"] += len(grown)
    COUNTS["ring growths with a straddling window"] += len(straddled)


def test_solo_state_covers_every_path():
    """Across the seeds above: every solo variant, speculative hits and misses, stand-downs, wraps and growths."""
    if COUNTS["seeds"] != len(SEEDS):
        pytest.skip("runs after all seeds of test_solo_state_across_calls")
    print(dict(COUNTS))
    for key in ("variant 2", "variant 3", "variant 4", "speculative hits", "speculative misses",
                "flag-4 stand-downs after a miss", "ring growths with a straddling window"):
        assert COUNTS[key] > 0, (key, dict(COUNTS))
    assert COUNTS["wrap seeds past 2^17 ids"] == sum(seed % 3 == 0 for seed in SEEDS), dict(COUNTS)
