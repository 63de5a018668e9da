"""The CPU half of the key-precision cases (tests/key_cases.py): the restatement walks each cluster exactly as the
Python model of UnsafePickServantFor does, the model shows the walk reaches the edge it is meant to, and the
restatement's results equal the reference's (fingerprints where the reference is not built)."""
import numpy as np
import pytest

import key_cases as K
from reference_results import check_reference
from yadcc_b200 import streams as S


def _replay(make_dispatcher, kind, name, with_self):
    d = make_dispatcher(kind)
    return S.Replayer(d, batch_heartbeats=True).run(K.key_stream(d, name, K.N_WALK, with_self))


@pytest.mark.parametrize("with_self", [False, True], ids=["walk", "self"])
@pytest.mark.parametrize("name", list(K.CLUSTERS))
def test_key_cluster_port_equals_model_and_reference(make_dispatcher, name, with_self):
    if not with_self:
        K.check_walk(name)
    mine = _replay(make_dispatcher, "port", name, with_self)
    status, pick, _, _, run = K.model_walk(name, with_self)
    g = mine[0]
    assert (g["status"] == status).all()
    ok = status == 2
    assert (g["servant_index"][ok] == pick[ok]).all()
    assert (g["task_id"][ok] == np.arange(int(ok.sum()))).all()
    assert (mine[1][:, 0] == run).all()
    check_reference(f"keys-{name}-{'self' if with_self else 'walk'}",
                    lambda: _replay(make_dispatcher, "ref", name, with_self), mine)
