"""The solo solve's direct launch and its wait on the request upload.  A solo solve waits for the copy stream only when
its call copied requests (a pageable array); staged and page-locked zero-copy solves carry no cross-stream dependency.
One CUDA handle alternates staged calls, pageable plain calls whose requests differ from the staged batch, page-locked
zero-copy calls, packed calls and a batch of another size class, and is compared with the CPU checker after every call.
A solve that read the request buffer before its upload landed would decide the staged batch instead, and its grants
would differ."""
import numpy as np
import pytest

from solve_lines import solves
from yadcc_b200 import STATUS_GRANTED, Servant, pack_requests
from yadcc_b200 import streams as S

pytestmark = pytest.mark.gpu

K = 4            # digests; servant i holds digest i % K, so every component is data-parallel (solo)
N_SERVANTS = 192
N = 1000         # one size class (1024) ...
N_OTHER = 3000   # ... and another (4096)
ROUND = ("staged", "pageable", "pinned", "packed", "staged", "pageable", "pinned", "packed", "other")
ROUNDS = 4


def _calls(d, seed):
    """(mode, requests) of every call, built on this handle's interned ids."""
    rng = np.random.default_rng(seed)
    dgs = [f"{0x50100000 + k:064x}" for k in range(K)]
    for i in range(N_SERVANTS):
        d.keep_servant_alive(Servant(f"{S.servant_ip(i)}:8335", None, [dgs[i % K]], 9, 64, 0, 256 << 30, 200 << 30, 24),
                             1e6, now=0.0)
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    ips = np.asarray([d.intern_ip(f"172.21.0.{i}") for i in range(200)], dtype=np.uint32)
    out = []
    for _ in range(ROUNDS):
        for mode in ROUND:
            n = N_OTHER if mode == "other" else N
            out.append((mode, S._requests(d, env[rng.integers(0, K, n)], ips[rng.integers(0, len(ips), n)], 8,
                                          expires_in_s=0.03, prefetch=rng.random(n) < 0.2)))
    return out


def _run(d, seed, capfd=None):
    """Grants and servant state after every call; the solve lines each call printed (capfd given)."""
    calls = _calls(d, seed)
    pinned, pinned16 = d.alloc_requests(N), d.alloc_requests16(N)
    trace, lines = [], []
    rng = np.random.default_rng(seed + 1)
    if capfd is not None:
        capfd.readouterr()
    for k, (mode, r) in enumerate(calls):
        now = 1.0 + 0.01 * k
        if mode == "staged":
            d.stage_requests(r)
            g = d.wait_for_staged_tasks(len(r), now)
        elif mode == "pinned":
            pinned[...] = r
            g = d.wait_for_starting_new_tasks(pinned, now)
        elif mode == "packed":
            pack_requests(r, pinned16)
            g = d.wait_for_starting_new_tasks_packed(pinned16, now)
        else:  # pageable: "pageable" and "other"
            g = d.wait_for_starting_new_tasks(np.ascontiguousarray(r), now)
        g = g.copy()
        trace += [g, d.servant_state().copy()]
        if capfd is not None:
            lines.append((mode, k % len(ROUND), k // len(ROUND), solves(capfd.readouterr().err),
                          d.last_solve_stats()["kernel_launches"]))
        granted = g["task_id"][g["status"] == STATUS_GRANTED]
        d.free_tasks(granted[rng.random(len(granted)) < 0.9].copy())  # (the rest expires a few calls later)
        d.on_expiration_timer(now=now + 0.005)
    return trace, lines


@pytest.mark.parametrize("graphs", [True, False], ids=["graph", "eager"])
def test_solo_solves_wait_for_their_upload_only(make_dispatcher, capfd, monkeypatch, graphs):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    d = make_dispatcher("cuda", graphs=graphs)
    got, lines = _run(d, 7, capfd)
    monkeypatch.delenv("YDSCHED_DEBUG")
    want, _ = _run(make_dispatcher("port"), 7)
    assert S.traces_equal(got, want), S.first_mismatch(got, want)
    assert all(len(ls) == 1 for _, _, _, ls, _ in lines), lines
    granted = [int((g["status"] == STATUS_GRANTED).sum()) for g in got[::2]]
    assert min(granted) > 0, granted
    # from the second round on, the batches after the first two of the 1024 size class are decided speculatively in ONE
    # launch, without a graph -- whichever way the requests came in
    steady = [(mode, ls[0], launches) for mode, pos, rnd, ls, launches in lines if rnd >= 1 and 3 <= pos < 8]
    assert {m for m, _, _ in steady} == {"staged", "pageable", "pinned", "packed"}
    for mode, x, launches in steady:
        assert (x["variant"], x["spec"], x["graph"], launches) == (4, 1, 0, 1), (mode, x, launches)
