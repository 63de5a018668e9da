"""In-flight task index: the CPU restatement (oracle/port.cc) against RunningTaskKeeper's
loops run literally over the verbatim TaskDispatcher/RunningTaskBookkeeper (oracle/_ref)."""
import pytest

from reference_results import check_reference
from running_index_cases import reference_test_case, run_suite


@pytest.mark.parametrize("seed", range(4))
def test_running_index_port_equals_reference(make_dispatcher, seed):
    check_reference(f"running-index-{seed}", lambda: run_suite(make_dispatcher("ref"), seed),
                    run_suite(make_dispatcher("port"), seed))


@pytest.mark.parametrize("backend", ["port", "ref"])
def test_running_task_keeper_reference_test(make_dispatcher, backend):
    first, second = reference_test_case(make_dispatcher(backend))
    assert first["found"].all() and list(first["servant_task_id"]) == [0, 1, 2]
    assert not second["found"].any()
