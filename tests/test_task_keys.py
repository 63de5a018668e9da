"""Cache keys and task digests derived from task descriptors (yd_derive_task_keys) and the pre-filtered solve that starts
from them (yd_derive_filter_and_wait_for_starting_new_tasks).

The keys are BLAKE3 over prefix || compiler digest || invocation arguments || source digest.  The CPU restatement (the
port) is checked byte for byte against the reference's own BLAKE3 on messages at every block and chunk boundary up to
the argument-length limit; the CUDA backend is checked against both, on the same cases and on the configs[3] descriptor
queue, and its descriptor pipeline against its key-based pipeline fed with keys derived on the host.

The checkers with the task keys are builds of their own: checkers/libydport_keys.so (the port) and
oracle/_ref/libydref_keys.so (the reference, where its sources are at hand).  The reference's results are kept as
fingerprints in tests/golden/task_keys_reference.json, so the comparison also runs where the reference is not built."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, cpu_backends
from reference_results import _same, fingerprint
from solve_lines import solves
from yadcc_b200 import REQ_DTYPE, STATUS_GRANTED, RunningTask, Servant, TaskDispatcher, TaskKeysError, TaskSources
from yadcc_b200 import _abi
from yadcc_b200 import streams as S

PORT_KEYS_LIB = ROOT / "checkers" / "libydport_keys.so"
REF_KEYS_LIB = ROOT / "oracle" / "_ref" / "libydref_keys.so"
STORE = ROOT / "tests" / "golden" / "task_keys_reference.json"
MAX = _abi.KEYS_MAX_ARGS_LEN
# compiler digests of every interned env id: a BLAKE3 hex digest, an empty one, a long one, bytes a client may send
ENVS = [f"{0xc0de0000 + k:064x}" for k in range(3)] + ["", "x" * 1500, "g++ 11.2 \x01\x7f"]
SRC_LEN = 64


@pytest.fixture
def keys_dispatcher(make_dispatcher):
    """Factory: keys_dispatcher('port'|'ref'|'cuda') -> a TaskDispatcher whose library exports the task keys."""
    made = []

    def factory(kind: str):
        if kind == "cuda":
            return make_dispatcher("cuda")
        if kind == "port" and not PORT_KEYS_LIB.exists():
            subprocess.check_call(["make", "-C", str(ROOT), "checkers/libydport_keys.so"])
        if kind == "ref" and not REF_KEYS_LIB.exists():
            pytest.skip("oracle/_ref/libydref_keys.so not built (needs the reference sources)")
        d = TaskDispatcher(str(PORT_KEYS_LIB if kind == "port" else REF_KEYS_LIB))
        made.append(d)
        return d

    yield factory
    for d in made:
        d.close()


def check_reference(key: str, run, mine) -> None:
    """`mine` equals the reference's result for `key`: in full where the reference is built (run() computes it;
    YD_WRITE_REFERENCE_RESULTS=1 then stores its fingerprint), and against the stored fingerprint everywhere."""
    stored = json.loads(STORE.read_text()) if STORE.exists() else {}
    if REF_KEYS_LIB.exists():
        live = run()
        assert _same(live, mine), f"{key}: differs from the reference"
        if os.environ.get("YD_WRITE_REFERENCE_RESULTS"):
            stored[key] = fingerprint(live)
            STORE.write_text(json.dumps(stored, indent=1, sort_keys=True) + "\n")
    assert key in stored, f"{key}: no stored reference result (build the reference, set YD_WRITE_REFERENCE_RESULTS=1)"
    assert fingerprint(mine) == stored[key], f"{key}: differs from the reference's stored result"


def _arg_lengths() -> list[int]:
    """0, 1, a block's edges, the lengths that put each message's end on a chunk's edge, and +-1 around 1..9 whole
    chunks and the limit."""
    out = {0, 1, 63, 64, 65, MAX - 1, MAX}
    for fixed in (16 + 64 + SRC_LEN, 4 + 64 + SRC_LEN, 16, 4):  # prefix + compiler digest + source digest
        for k in (1, 2, 3, 4, 5, 8, 9):
            out.update(k * 1024 - fixed + d for d in (-1, 0, 1))
    for k in (1, 2, 3, 4, 5, 8, 9, 255):
        out.update(k * 1024 + d for d in (-1, 0, 1))
    return sorted(x for x in out if 0 <= x <= MAX)


def _boundary_case(d, src_len: int = SRC_LEN, seed: int = 5):
    """Requests over every (argument length, env id) pair, arguments of arbitrary bytes (NUL included)."""
    env = [d.intern_env(e) for e in ENVS]
    rng = np.random.default_rng(seed)
    lens = _arg_lengths()
    args = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in lens]
    idx = np.arange(len(lens) * len(env)) % len(lens)
    reqs = np.zeros(len(idx), dtype=REQ_DTYPE)
    reqs["env_id"] = np.asarray(env, dtype=np.uint32)[np.arange(len(idx)) // len(lens)]
    sd = np.frombuffer(rng.bytes(len(idx) * src_len), dtype=np.uint8).reshape(len(idx), src_len).copy()
    sd[::7] = 0  # NUL-filled records too
    return reqs, TaskSources.of(args, idx, sd)


def _derive(kind, keys_dispatcher, src_len=SRC_LEN):
    d = keys_dispatcher(kind)
    reqs, src = _boundary_case(d, src_len)
    return d.derive_task_keys(reqs, src)


# ---- CPU ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("src_len", [SRC_LEN, 0])
def test_port_keys_match_reference_at_every_boundary(keys_dispatcher, src_len):
    keys, digests = _derive("port", keys_dispatcher, src_len)
    assert keys.shape[1] == 81 and digests.shape[1] == 64
    assert (keys[:, :17] == np.frombuffer(b"yadcc-cxx2-entry-", dtype=np.uint8)).all()
    hexchars = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    assert np.isin(keys[:, 17:], hexchars).all() and np.isin(digests, hexchars).all()
    check_reference(f"task_keys/boundaries/src{src_len}", lambda: _derive("ref", keys_dispatcher, src_len), (keys, digests))


def test_split_between_pieces_does_not_matter(keys_dispatcher):
    """BLAKE3 hashes the plain concatenation: "cxx2" || "" || "abc" || "" == "cxx2" || "" || "a" || "bc"."""
    d = keys_dispatcher("port")
    reqs = np.zeros(1, dtype=REQ_DTYPE)
    reqs["env_id"] = d.intern_env("")
    a = d.derive_task_keys(reqs, TaskSources.of([b"abc"], [0], np.zeros((1, 0), np.uint8)), cache_keys=False)[1]
    b = d.derive_task_keys(reqs, TaskSources.of([b"a"], [0], np.frombuffer(b"bc", np.uint8).reshape(1, 2)),
                           cache_keys=False)[1]
    assert (a == b).all()


def _errors_case(d):
    env = d.intern_env(ENVS[0])
    reqs = np.zeros(3, dtype=REQ_DTYPE)
    reqs["env_id"] = env
    sd = np.full((3, SRC_LEN), ord("s"), dtype=np.uint8)
    return env, reqs, sd


def _expect_error(d, reqs, src, code):
    keys = np.full((len(reqs), 81), 0xAB, dtype=np.uint8)
    dg = np.full((len(reqs), 64), 0xCD, dtype=np.uint8)
    f = src.struct()
    rc = d._lib.yd_derive_task_keys(d._h, reqs.ctypes.data, len(reqs), C.byref(f), keys.ctypes.data, dg.ctypes.data)
    assert rc == code
    assert (keys == 0xAB).all() and (dg == 0xCD).all(), "an error wrote output"
    with pytest.raises(TaskKeysError) as e:
        d.derive_task_keys(reqs, src)
    assert e.value.code == code


def _check_errors(d):
    env, reqs, sd = _errors_case(d)
    ok = TaskSources.of([b"-c", b"x" * MAX], [0, 1, 0], sd)
    d.derive_task_keys(reqs, ok)  # the limit itself is taken
    _expect_error(d, reqs, TaskSources.of([b"-c", b"x" * (MAX + 1)], [0, 0, 0], sd), _abi.KEYS_TOO_LONG)
    _expect_error(d, reqs, TaskSources.of([b"-c"], [0, 1, 0], sd), _abi.KEYS_BAD_ARGS_INDEX)
    bad_env = reqs.copy()
    bad_env["env_id"][2] = env + 100
    _expect_error(d, bad_env, ok, _abi.KEYS_UNKNOWN_ENV)
    long_sd = np.zeros((3, _abi.KEYS_MAX_DIGEST_LEN + 1), dtype=np.uint8)
    _expect_error(d, reqs, TaskSources.of([b"-c"], [0, 0, 0], long_sd), _abi.KEYS_TOO_LONG)
    backwards = TaskSources.of([b"-c", b"-O2"], [0, 1, 0], sd)
    backwards.args_offsets[1] = 9  # past the end offset 5
    _expect_error(d, reqs, backwards, _abi.KEYS_BAD_SOURCES)


@pytest.mark.parametrize("kind", cpu_backends())
def test_bad_input_is_refused_with_nothing_written(keys_dispatcher, kind):
    _check_errors(keys_dispatcher(kind))


def _cluster(d, n_servants=48, envs=ENVS[:3]):
    for i in range(n_servants):
        d.keep_servant_alive(Servant(f"{S.servant_ip(i)}:8335", None, [envs[i % len(envs)]], 9, 16, 0, 256 << 30,
                                     200 << 30, 8), 1e6, now=0.0)
    return np.asarray([d.intern_env(e) for e in envs], dtype=np.uint32)


def _queue(d, env, n, seed):
    """n requests over 200 TUs (some repeat within the queue) with their descriptors."""
    rng = np.random.default_rng(seed)
    ips = np.asarray([d.intern_ip(f"172.22.0.{i}") for i in range(50)], dtype=np.uint32)
    tu = rng.integers(0, 200, n)
    reqs = S._requests(d, env[tu % len(env)], ips[rng.integers(0, len(ips), n)], 8, expires_in_s=5.0)
    r2 = np.random.default_rng(99)
    args = [bytes(r2.integers(32, 127, int(m), dtype=np.uint8)) for m in np.geomspace(50, 5000, 12).astype(int)]
    tu_src = np.frombuffer(r2.bytes(200 * SRC_LEN), dtype=np.uint8).reshape(200, SRC_LEN)
    return reqs, TaskSources.of(args, (np.arange(200) % len(args))[tu], tu_src[tu])


def _filter_state(d, env, host_keys):
    """Bloom filter holding the cache keys of a third of the first queue's requests; running tasks listing the task
    digests of another third.  host_keys: the dispatcher whose derive_task_keys makes the keys."""
    reqs, src = _queue(d, env, 400, 1)
    keys, digests = host_keys.derive_task_keys(reqs, src)
    d.bloom_reset(1 << 16, 4)
    d.bloom_add(keys[::3])
    early = d.wait_for_starting_new_tasks(reqs[:60].copy(), 0.5)
    by = {}
    for j, g in enumerate(early):
        if g["status"] == STATUS_GRANTED:
            by.setdefault(int(g["servant_index"]), []).append(
                RunningTask(j + 1, int(g["task_id"]), d.servant_location(int(g["servant_index"])), bytes(digests[1 + 3 * j]).decode()))
    d.notify_servants_running_tasks([(d.servant_location(k), v) for k, v in by.items()])
    d.running_index_refresh()


def _descriptor_pipeline(d, stages, host_keys=None):
    """Several calls of the descriptor pipeline with frees and ticks between them; host_keys given: the key-based
    pipeline fed with keys host_keys derives instead."""
    env = _cluster(d)
    if host_keys is not None and host_keys is not d:  # (the same intern table: both handles are fresh)
        assert [host_keys.intern_env(e) for e in ENVS[:3]] == list(env)
    _filter_state(d, env, host_keys or d)
    out = []
    for k in range(4):
        reqs, src = _queue(d, env, 500 + 37 * k, 2 + k)
        now = 1.0 + 0.1 * k
        if host_keys is None:
            v, h, g = d.derive_filter_and_wait_for_starting_new_tasks(reqs, src, stages, now)
        else:
            keys, digests = host_keys.derive_task_keys(reqs, src)
            v, h, g = d.filter_and_wait_for_starting_new_tasks(reqs, keys if stages & 1 else None,
                                                               digests if stages & 2 else None, now)
        again = d.wait_for_staged_tasks(len(g), now + 0.01) if len(g) else g  # the staged queue afterwards
        out += [v.copy(), h.copy(), g.copy(), again.copy(), d.servant_state().copy()]
        granted = np.concatenate([g, again])
        granted = granted["task_id"][granted["status"] == STATUS_GRANTED]
        d.free_tasks(granted[::2].copy())
        d.on_expiration_timer(now=now + 0.05)
    return out


@pytest.mark.parametrize("stages", [3, 1, 2, 0], ids=["both", "cache", "dedupe", "none"])
def test_port_pipeline_is_derive_then_filter_call_on_reference(keys_dispatcher, stages):
    mine = _descriptor_pipeline(keys_dispatcher("port"), stages)
    assert any((v == _abi.FILTER_CACHE_HIT).any() for v in mine[0::5]) == bool(stages & 1)
    assert any((v == _abi.FILTER_JOINED).any() for v in mine[0::5]) == bool(stages & 2)

    def ref():
        d = keys_dispatcher("ref")
        return _descriptor_pipeline(d, stages, host_keys=d)

    check_reference(f"task_keys/pipeline/stages{stages}", ref, mine)


def test_refused_pipeline_decides_nothing_and_keeps_the_staged_queue(keys_dispatcher):
    d = keys_dispatcher("port")
    env = _cluster(d)
    reqs, src = _queue(d, env, 100, 3)
    d.stage_requests(reqs[:10].copy())
    bad = TaskSources.of([b"-c"], np.full(100, 1), src.source_digests)
    with pytest.raises(TaskKeysError):
        d.derive_filter_and_wait_for_starting_new_tasks(reqs, bad, 0, 1.0)
    assert d.num_tasks() == 0
    assert (d.wait_for_staged_tasks(10, 1.0)["status"] == STATUS_GRANTED).all()


def test_task_sources_struct_layout():
    f = _abi.yd_task_sources
    assert C.sizeof(f) == 56
    assert [getattr(f, x).offset for x in ("args", "args_offsets", "n_args", "args_index", "source_digests",
                                            "source_digest_len", "source_digest_stride")] == [0, 8, 16, 24, 32, 40, 48]


# ---- GPU ------------------------------------------------------------------------------------------------------

def _host_lib(keys_dispatcher):
    return keys_dispatcher("ref" if REF_KEYS_LIB.exists() else "port")


@pytest.mark.gpu
@pytest.mark.parametrize("src_len", [SRC_LEN, 0])
def test_cuda_keys_match_port_and_reference(keys_dispatcher, src_len):
    got = _derive("cuda", keys_dispatcher, src_len)
    want = _derive("port", keys_dispatcher, src_len)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    check_reference(f"task_keys/boundaries/src{src_len}", lambda: _derive("ref", keys_dispatcher, src_len), got)
    # one kind of output at a time
    d = keys_dispatcher("cuda")
    reqs, src = _boundary_case(d, src_len)
    assert d.derive_task_keys(reqs, src, task_digests=False)[1] is None
    assert (d.derive_task_keys(reqs, src, task_digests=False)[0] == want[0]).all()
    assert (d.derive_task_keys(reqs, src, cache_keys=False)[1] == want[1]).all()


@pytest.mark.gpu
def test_cuda_keys_on_the_configs3_descriptor_queue(keys_dispatcher):
    src = S.config3_task_sources(100_000)
    out = []
    for kind in ("cuda", "port"):
        d = keys_dispatcher(kind)
        w = S.config2(100_000, 2000, 8, seed=42, variant="mod")
        w.register(d)
        out.append(d.derive_task_keys(w.build_requests(d), src))
    assert (out[0][0] == out[1][0]).all() and (out[0][1] == out[1][1]).all()
    assert len(set(map(bytes, out[0][1]))) > 6124  # (TUs meet different compilers as the trace loops)


@pytest.mark.gpu
def test_cuda_refuses_bad_input_with_nothing_written(keys_dispatcher):
    _check_errors(keys_dispatcher("cuda"))
    d = keys_dispatcher("cuda")
    env = _cluster(d)
    reqs, src = _queue(d, env, 100, 3)
    d.stage_requests(reqs[:10].copy())
    with pytest.raises(TaskKeysError):
        d.derive_filter_and_wait_for_starting_new_tasks(reqs, TaskSources.of([b"-c"], np.full(100, 1), src.source_digests), 0, 1.0)
    assert d.num_tasks() == 0
    assert (d.wait_for_staged_tasks(10, 1.0)["status"] == STATUS_GRANTED).all()


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [3, 1, 2, 0], ids=["both", "cache", "dedupe", "none"])
def test_cuda_descriptor_pipeline_equals_key_pipeline_with_host_keys(keys_dispatcher, stages):
    got = _descriptor_pipeline(keys_dispatcher("cuda"), stages)
    want = _descriptor_pipeline(keys_dispatcher("cuda"), stages, host_keys=_host_lib(keys_dispatcher))
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype and a.shape == b.shape and (a == b).all(), f"call {i // 5}, item {i % 5}"
    # and what the port computes for the whole pipeline
    port = _descriptor_pipeline(keys_dispatcher("port"), stages)
    assert all((a == b).all() for a, b in zip(got, port))
    # h2d_bytes counts what was uploaded: against the key-based call on the same queue, the descriptors instead of the
    # keys (and, on the first derivation, the env table)
    d = keys_dispatcher("cuda")
    env = _cluster(d)
    d.bloom_reset(1 << 16, 4)
    reqs, src = _queue(d, env, 1000, 4)
    d.derive_filter_and_wait_for_starting_new_tasks(reqs, src, stages, 1.0)
    desc = d.last_solve_stats()
    assert desc["decisions"] == 1000 and desc["prep_ms"] > 0
    keys, digests = d.derive_task_keys(reqs, src)
    d.filter_and_wait_for_starting_new_tasks(reqs, keys if stages & 1 else None, digests if stages & 2 else None, 1.1)
    key = d.last_solve_stats()
    descriptors = int(src.args_offsets[-1]) + 8 * len(src.args_offsets) + 4 * 1000 + src.source_digests.nbytes
    env_table = sum(len(e) for e in ENVS[:3]) + 4 * 4
    expect = (descriptors + env_table - (81 * 1000 if stages & 1 else 0) - (64 * 1000 if stages & 2 else 0)) if stages else 0
    assert int(desc["h2d_bytes"]) - int(key["h2d_bytes"]) == expect


@pytest.mark.gpu
def test_cuda_env_table_follows_heartbeats_and_import(keys_dispatcher):
    d, port = keys_dispatcher("cuda"), keys_dispatcher("port")
    for x in (d, port):
        _cluster(x)
    reqs, src = _queue(d, np.asarray([0, 1, 2], np.uint32), 300, 6)
    assert all((a == b).all() for a, b in zip(d.derive_task_keys(reqs, src), port.derive_task_keys(reqs, src)))
    # a heartbeat brings new digests after the table went to the device
    for x in (d, port):
        x.keep_servant_alive(Servant("10.9.9.9:8335", None, ["new-compiler-a", ENVS[4]], 9, 16, 0, 256 << 30, 200 << 30, 8),
                             1e6, now=0.5)
    new = [d.intern_env(e) for e in ("new-compiler-a", ENVS[4])]
    assert new == [port.intern_env(e) for e in ("new-compiler-a", ENVS[4])]
    reqs["env_id"] = np.asarray(new * 150, np.uint32)
    assert all((a == b).all() for a, b in zip(d.derive_task_keys(reqs, src), port.derive_task_keys(reqs, src)))
    # a fresh handle that imports the state derives with the imported intern table
    blob = d.export_state(1.0)
    d2 = keys_dispatcher("cuda")
    d2.import_state(blob, 1.0)
    assert all((a == b).all() for a, b in zip(d2.derive_task_keys(reqs, src), port.derive_task_keys(reqs, src)))


@pytest.mark.gpu
def test_solo_solve_after_a_derivation_stays_speculative(keys_dispatcher, capfd, monkeypatch):
    monkeypatch.setenv("YDSCHED_DEBUG", "1")
    d = keys_dispatcher("cuda")
    monkeypatch.delenv("YDSCHED_DEBUG")
    dgs = [f"{0x50200000 + k:064x}" for k in range(4)]
    for i in range(192):
        d.keep_servant_alive(Servant(f"{S.servant_ip(i)}:8335", None, [dgs[i % 4]], 9, 64, 0, 256 << 30, 200 << 30, 24),
                             1e6, now=0.0)
    env = np.asarray([d.intern_env(x) for x in dgs], dtype=np.uint32)
    ips = np.asarray([d.intern_ip(f"172.23.0.{i}") for i in range(100)], dtype=np.uint32)
    rng = np.random.default_rng(8)
    d.bloom_reset(1 << 16, 4)
    _, src = _queue(d, env, 1000, 9)
    variants = []
    for k in range(8):
        now = 1.0 + 0.01 * k
        r = S._requests(d, env[rng.integers(0, 4, 1000)], ips[rng.integers(0, 100, 1000)], 8, expires_in_s=0.005)
        if k == 0:  # the pipeline's own buffers are in place from here on
            _, _, g = d.derive_filter_and_wait_for_starting_new_tasks(r.copy(), src, 3, now)
            d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED].copy())
        d.derive_task_keys(r, src)
        capfd.readouterr()
        g = d.wait_for_starting_new_tasks(r.copy(), now + 0.007)
        assert (g["status"] == STATUS_GRANTED).any()
        variants.append([(x["variant"], x["spec"]) for x in solves(capfd.readouterr().err)])
        d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED].copy())
        d.on_expiration_timer(now=now + 0.009)
    assert all(v == [(4, 1)] for v in variants[3:]), variants


def test_keys_header_is_exported_by_every_build_that_has_it():
    """include/ydkeys.h is declared one-to-one in _abi.KEYS_PROTOTYPES and exported by the CUDA library and the
    checkers' key builds."""
    from test_abi import header_symbols

    names = header_symbols("ydkeys.h")
    assert names == sorted(name for name, _, _ in _abi.KEYS_PROTOTYPES)
    for lib in (ROOT / "yadcc_b200" / "libydsched.so", PORT_KEYS_LIB, REF_KEYS_LIB):
        if lib == REF_KEYS_LIB and not lib.exists():
            continue
        h = C.CDLL(str(lib))
        assert all(hasattr(h, name) for name in names), lib
