"""The speculative solo solve's one-hop lookups (fused.cuh, classes.cuh: kept_class): a request reads its digest's word
of the kept class table (kept_env) and its IP's component mask (ip_comp_mask), and a slot reads its servant's kept class
(kept_sv).  The cases those tables add: a digest of a component that holds another digest's class, a digest of a
component without any class, and requestor IPs whose servants sit in a component beyond the mask's 64 bits (the IP CSR
is walked instead) -- each replayed through the CUDA backend and compared with the CPU checker, with the speculative
outcome of every probe batch read from the YDSCHED_DEBUG solve lines."""
import numpy as np
import pytest

from yadcc_b200 import Servant
from yadcc_b200 import streams as S
from solve_lines import solves

pytestmark = pytest.mark.gpu

N = 1000  # requests per batch (one size class: the kept class table sits behind res[], whose size follows it)


def _servant(i: int, digests: list) -> Servant:
    return Servant(f"{S.servant_ip(i)}:8335", None, digests, 10, 64, 0, 256 << 30, 200 << 30, 24)


class _Batches:
    def __init__(self, d, ev, seed):
        self.d, self.ev, self.rng, self.now, self.kinds = d, ev, np.random.default_rng(seed), 0.001, []
        self.outside = np.asarray([d.intern_ip(f"172.16.2.{i}") for i in range(100)], dtype=np.uint32)

    def add(self, kind, env, ips=None):
        """One batch of requests for the digest ids `env` (cycled), from `ips` or from outside the cluster."""
        rng = self.rng
        e = np.asarray(env, dtype=np.uint32)[rng.integers(0, len(env), N)]
        if ips is None:
            ips = self.outside[rng.integers(0, len(self.outside), N)]
        mv = np.full(N, 8, np.uint32)
        self.ev.append(("wait", self.now, S._requests(self.d, e, ips, mv, expires_in_s=15.0, prefetch=rng.random(N) < 0.2)))
        self.ev.append(("state",))
        self.ev.append(("free_frac", int(rng.integers(1 << 30)), 0.5))
        self.ev.append(("tick", self.now + 0.005))
        self.now += 0.01
        self.kinds.append(kind)


def _digests(k):
    return [f"{0x6b000000 + i:064x}" for i in range(k)]


def _stream_shared_components(d):
    """Component 0 holds digests A and B, component 1 digest C, component 2 digest D.  The steady batches ask for A and
    C, so the kept table has a class for components 0 and 1 only; probes ask for B (its component holds A's class) and
    for D (its component holds no class): both must miss and be replayed."""
    dg = _digests(4)
    ev = []
    for i in range(96):
        ev.append(("hb", 0.0, _servant(i, [dg[0], dg[1]] if i % 3 == 0 else [dg[2 + i % 3 - 1]]), 100.0))
    env = [d.intern_env(x) for x in dg]
    b = _Batches(d, ev, seed=5)
    steady = [env[0], env[2]]
    for _ in range(4):
        b.add("steady", steady)
    b.add("probe-other-digest", steady + [env[1]])
    for _ in range(4):
        b.add("steady", steady)
    b.add("probe-no-class", steady + [env[3]])
    for _ in range(4):
        b.add("steady", steady)
    return S.Stream("kept-shared-components", ev), b.kinds


def _stream_wide_components(d):
    """80 components, one digest each (servant i holds digest i % 80, so component c is digest c's).  The steady batches
    ask for digests 5, 70 and 71; probes come from the IP of servant 70 (component 70, beyond the IP mask's 64 bits):
    asking for digest 70 they are self-requests and must miss; asking for digests 5 and 71 they are not."""
    dg = _digests(80)
    ev = [("hb", 0.0, _servant(i, [dg[i % 80]]), 100.0) for i in range(160)]
    env = [d.intern_env(x) for x in dg]
    own = d.intern_ip(S.servant_ip(70))
    b = _Batches(d, ev, seed=6)
    steady = [env[5], env[70], env[71]]
    for _ in range(4):
        b.add("steady", steady)
    b.add("probe-other-components", [env[5], env[71]], ips=np.full(N, own, np.uint32))
    for _ in range(3):
        b.add("steady", steady)
    b.add("probe-self", steady, ips=np.where(np.arange(N) % 10 == 0, own, b.outside[np.arange(N) % 100]))
    for _ in range(4):
        b.add("steady", steady)
    return S.Stream("kept-wide-components", ev), b.kinds


@pytest.mark.parametrize("make_stream", [_stream_shared_components, _stream_wide_components], ids=["shared", "wide"])
@pytest.mark.parametrize("packed", [True, False], ids=["packed", "plain"])
def test_kept_lookups_equal_oracle(make_dispatcher, monkeypatch, capfd, make_stream, packed):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    traces = {}
    for kind in ("cuda", "port"):
        d = make_dispatcher(kind)
        stream, kinds = make_stream(d)
        traces[kind] = S.Replayer(d, pinned=(kind == "cuda"), packed=(packed and kind == "cuda")).run(stream)
        d.close()
    assert S.traces_equal(traces["cuda"], traces["port"]), S.first_mismatch(traces["cuda"], traces["port"])
    lines = [x for x in solves(capfd.readouterr().err) if x["n"] == N]
    assert len(lines) == len(kinds), (len(lines), len(kinds))
    spec = {k: [x["spec"] for x, kk in zip(lines, kinds) if kk == k] for k in set(kinds)}
    assert 1 in spec["steady"], spec  # the steady stretches were decided speculatively
    for k, v in spec.items():
        if k in ("probe-other-digest", "probe-no-class", "probe-self"):
            assert v == [2], (k, spec)  # speculated, missed, replayed
        elif k == "probe-other-components":
            assert v == [1], (k, spec)  # requests from a servant's IP for other components: a hit
