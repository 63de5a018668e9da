"""SchedulerServiceImpl::WaitForStartingTask's request expansion
(scheduler_service_impl.cc:209-271) through yd_wait_for_starting_task_rpcs: the batched
implementation (include/ydsched_rpc_impl.inc, here over the CPU restatement) against the
reference's literal loops over the verbatim TaskDispatcher (oracle/ref_harness.cc)."""
import numpy as np
import pytest

from reference_results import check_reference
from rpc_cases import run_rpc_stream
from yadcc_b200 import Servant, _abi


@pytest.mark.parametrize("seed", range(40))
def test_rpc_expansion_port_equals_reference(make_dispatcher, seed):
    check_reference(f"rpc-expansion-{seed}", lambda: run_rpc_stream(make_dispatcher("ref"), seed),
                    run_rpc_stream(make_dispatcher("port"), seed))


@pytest.mark.parametrize("backend", ["port", "ref"])
def test_rpc_status_quirks(make_dispatcher, backend):
    """Hand-checked against scheduler_service_impl.cc: :242-246 (unknown environment on an
    immediate request -> 1006), :260-262 + :266-270 (unknown environment on a prefetch-only
    RPC -> 1001), :221-226 (limits -> 1004, nothing attempted), grants are a prefix."""
    d = make_dispatcher(backend)
    d.keep_servant_alive(Servant("10.6.1.1:8335", None, ["d"], 8, 8, 0, 0, 64 << 30, 3), 10.0, now=0.0)
    rpcs = np.zeros(6, dtype=_abi.RPC_WAIT_DTYPE)
    rpcs["requestor_ip"] = d.intern_ip("10.9.9.9")
    rpcs["next_keep_alive_ns"] = 15_000_000_000
    rpcs["env_id"] = [d.intern_env(x) for x in ["nope", "nope", "d", "d", "d", "d"]]
    rpcs["immediate_reqs"] = [1, 0, 2, 1, 1, 2]
    rpcs["prefetch_reqs"] = [1, 2, 0, 0, 1, 2]
    rpcs["milliseconds_to_wait"] = [0, 0, 0, 10001, 0, 0]
    res, grants = d.wait_for_starting_task_rpcs(rpcs, now=0.0)
    assert res["status"].tolist() == [1006, 1001, 0, 1004, 0, 1001]
    assert res["n_grants"].tolist() == [0, 0, 2, 0, 1, 0]  # 3 slots: two, then one, then none
    assert grants["task_id"].tolist() == [0, 1, 2]
