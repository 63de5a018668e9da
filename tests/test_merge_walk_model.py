"""The plain model of the merge solver's walk (merge_walk_model.py) on every hand-back case (merge_cases.py): each case
reaches exactly the edge it names, and where no blocking pair forms the model's decisions are the CPU restatement's
(and the reference's where it is built) -- so the GPU cases compare against a walk whose side of every rule is known.
"""
import functools

import numpy as np
import pytest

import merge_cases as M
import merge_walk_model as W
from conftest import REF_LIB, _ensure_port
from yadcc_b200 import STATUS_GRANTED, TaskDispatcher
from yadcc_b200 import streams as S


@functools.lru_cache(maxsize=None)
def _walk(name):
    c = M.ALL[name]
    return W.walk(c.servants, c.reqs)


def _checkers():
    return [str(_ensure_port())] + ([str(REF_LIB)] if REF_LIB.exists() else [])


@pytest.mark.parametrize("name", list(M.ALL))
def test_case_reaches_its_edge(name):
    c, w = M.ALL[name], _walk(name)
    assert c.edge(w), (name, w.pend, w.skip, w.blocking)
    assert bool(w.blocking) == bool(c.back & M.BACK_CHECK)
    assert (w.pend > M.MERGE_PEND) == bool(c.back & M.BACK_PEND)
    assert (w.skip > M.MERGE_SKIP) == bool(c.back & M.BACK_SKIP)
    if name in M.SHARDED:
        assert (w.margin() >= M.RQ_MARGIN) == (name == "margin-1024")
    # a pass can never extend a run: the slot that made the run took the request right behind it
    assert w.merges == 0


@pytest.mark.parametrize("name", list(M.ALL))
def test_model_equals_checkers(name):
    c, w = M.ALL[name], _walk(name)
    for lib in _checkers():
        d = TaskDispatcher(lib)
        try:
            g = S.Replayer(d, batch_heartbeats=True).run(M.stream(d, c))[0]
        finally:
            d.close()
        if w.blocking:
            # the walk differs from the sequential fold exactly at a blocking pair: the request takes its own servant
            q = w.blocking[0]
            assert g["status"][q] == STATUS_GRANTED and g["servant_index"][q] != w.pick[q]
            continue
        assert (g["status"] == np.asarray(w.status)).all(), lib
        ok = g["status"] == STATUS_GRANTED
        assert (g["servant_index"][ok] == np.asarray(w.pick)[ok]).all(), lib
