"""The bloom pre-filter's CPU restatement (oracle/port.cc: own XXH64) against flare's
SaltedBloomFilter + the vendored xxHash compiled verbatim (oracle/_ref)."""
import numpy as np
import pytest

from bloom_cases import run_bloom_suite, tu_keys
from reference_results import check_reference


@pytest.mark.parametrize("seed", range(3))
def test_bloom_port_equals_reference(make_dispatcher, seed):
    check_reference(f"bloom-{seed}", lambda: run_bloom_suite(make_dispatcher("ref"), seed),
                    run_bloom_suite(make_dispatcher("port"), seed))


@pytest.mark.parametrize("backend", ["port", "ref"])
def test_bloom_behaviour(make_dispatcher, backend):
    """The reference's own behavioural checks (flare/base/experimental/bloom_filter_test.cc:
    44-73, yadcc/cache/bloom_filter_generator_test.cc:24-75): no false negatives, few false
    positives at yadcc's geometry; plus XXH64("") = 0xEF46DB3751D8E999 seen through a
    1-hash filter with an empty... (salted) key is covered by byte equality above."""
    d = make_dispatcher(backend)
    keys = tu_keys(4000)
    d.bloom_reset()
    d.bloom_add(keys[:2000])
    got = d.bloom_possibly_contains(keys)
    assert got[:2000].all()
    assert got[2000:].sum() <= 2  # p ~ 1e-5 at this load
    assert len(d.bloom_bytes()) == (1 << 25) // 8
