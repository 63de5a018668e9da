"""The CPU restatement (oracle/port.cc) against the reference compiled verbatim
(oracle/_ref) on seeded event streams -- fingerprints of its results where it is not
built (tests/reference_results.py) -- plus the committed golden digests that were
generated from the verbatim build (tests/golden/make_golden.py)."""
import json
import os
from pathlib import Path

import numpy as np
import pytest

from reference_results import check_reference
from yadcc_b200 import streams as S

GOLDEN = Path(__file__).parent / "golden"


def _replay(make_dispatcher, kind, build):
    d = make_dispatcher(kind)
    return S.Replayer(d).run(build(d))


def _port_equals_reference(make_dispatcher, key, build):
    check_reference(key, lambda: _replay(make_dispatcher, "ref", build), _replay(make_dispatcher, "port", build))


@pytest.mark.parametrize("seed", range(60))
def test_fuzz_port_equals_reference(make_dispatcher, seed):
    _port_equals_reference(make_dispatcher, f"fuzz-{seed}",
                           lambda d: S.fuzz_stream(d, seed, n_servants=8 + seed % 30, wide=(seed % 5 == 0)))


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 5, 11])
def test_solo_stream_port_equals_reference(make_dispatcher, seed):
    """The solo-path streams of tests/test_solo_state.py: version gating, servant churn, shared hosts, zombies, the
    lease ring past 2^17 ids (seeds 0, 3) with a pinned window (seed 0) -- the reference's behaviour, not the
    restatement's."""
    _port_equals_reference(make_dispatcher, f"solo-{seed}", lambda d: S.solo_stream(d, seed))


@pytest.mark.parametrize("name", ["cfg1", "cfg2-mod-small", "cfg2-random-small", "cfg3-small"])
def test_configs_port_equals_reference(make_dispatcher, name):
    _port_equals_reference(make_dispatcher, f"config-{name}", lambda d: S.named_stream(name, d))


def test_port_matches_committed_golden_digests(make_dispatcher):
    """Golden digests come from the reference itself (oracle/_ref), so this pins
    the restatement even where /root/reference is absent."""
    golden = json.loads((GOLDEN / "digests.json").read_text())
    huge = () if os.environ.get("YD_GOLDEN_HUGE") else ("cfg3", "cfg5-1m")  # minutes each on a CPU: opt-in here, always on the GPU
    for name, want in golden["streams"].items():
        if name in huge:
            continue
        d = make_dispatcher("port")
        tr = S.Replayer(d).run(S.named_stream(name, d))
        assert S.trace_digest(tr) == want["sha256"], name
        d.close()


def test_port_matches_committed_cfg1_vectors(make_dispatcher):
    z = np.load(GOLDEN / "cfg1_reference.npz")
    d = make_dispatcher("port")
    tr = S.Replayer(d).run(S.named_stream("cfg1", d))
    g = tr[0]
    assert (g["status"] == z["status"]).all()
    assert (g["task_id"] == z["task_id"]).all()
    assert (g["servant_index"] == z["servant_index"]).all()


@pytest.mark.parametrize("kind", ["port", "ref"])
@pytest.mark.parametrize("seed", range(0, 40, 3))
def test_batched_heartbeats_equal_single_calls(make_dispatcher, kind, seed):
    """yd_keep_servants_alive / yd_notify_servants_running_tasks are defined as the loop over the
    single-servant calls: replaying a stream with its heartbeat runs batched changes nothing."""
    traces = []
    for batched in (False, True):
        d = make_dispatcher(kind)
        traces.append(S.Replayer(d, batch_heartbeats=batched).run(S.fuzz_stream(d, seed, n_servants=8 + seed % 30)))
        d.close()
    assert S.traces_equal(*traces), S.first_mismatch(*traces)


@pytest.mark.parametrize("seed", [0, 7, 13, 21])
def test_dump_internals_port_equals_reference(make_dispatcher, seed):
    """TaskDispatcher::DumpInternals (task_dispatcher.cc:538-614): the per-servant rows and the five summary fields
    the reference's own function produces (written out by the harness from its Json::Value) against the
    restatement's -- after a stream that leaves servants in every state (full, low memory, not accepting, expired)."""
    def dump(kind):
        d = make_dispatcher(kind)
        assert d.dump_internals() == {"servants_up": 0, "running_tasks": 0, "capacity": 0, "capacity_available": 0,
                                      "capacity_unavailable": 0}
        S.Replayer(d).run(S.fuzz_stream(d, seed, n_servants=10 + seed))
        return d.dump_internals()

    mine = dump("port")
    check_reference(f"dump-internals-{seed}", lambda: dump("ref"), mine)
    assert len(mine.get("servants", [])) == mine["servants_up"]
