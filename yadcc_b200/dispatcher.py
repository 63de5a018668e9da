"""Host-side mirror of the reference's `TaskDispatcher` public interface.

Same method names, argument meaning and error behaviour as
yadcc/scheduler/task_dispatcher.h:120-181, so that tests read like the
reference's own (yadcc/scheduler/task_dispatcher_test.cc).  Differences, all
forced by deterministic replay (SURVEY.md 8(b)):

* time is an explicit ``now`` argument (seconds, float or int nanoseconds via
  ``now_ns=``) instead of ``flare::ReadCoarseSteadyClock()``;
* the 1 Hz expiration timer is fired by the caller (``on_expiration_timer``);
* ``wait_for_starting_new_task`` never blocks: ``timeout`` is accepted for
  signature parity but a request that finds no free servant fails with
  ``WaitStatus.Timeout`` at once (zero-wait discipline);
* the batched ``wait_for_starting_new_tasks`` is the hot path: *n* sequential
  calls in one C-ABI crossing.

All computation happens behind the C ABI (include/ydsched.h); this file only
marshals arguments.
"""
from __future__ import annotations

import ctypes as C
import enum
import json
from dataclasses import dataclass, field
from typing import Iterable, Sequence

import numpy as np

from . import _abi
from ._abi import GRANT_DTYPE, REQ_DTYPE, SERVANT_STATE_DTYPE


class WaitStatus(enum.IntEnum):
    """task_dispatcher.h:41-44."""

    EnvironmentNotFound = 0
    Timeout = 1


@dataclass
class TaskAllocation:
    """task_dispatcher.h:69-77."""

    task_id: int
    servant_location: str


@dataclass
class Servant:
    """ServantPersonality, task_dispatcher.h:80-116."""

    observed_location: str
    reported_location: str | None = None
    environments: Sequence[str] = ()
    version: int = 0
    num_processors: int = 0
    current_load: int = 0
    total_memory_in_bytes: int = 0
    memory_available_in_bytes: int = 0
    max_tasks: int = 0
    priority: int = _abi.PRIORITY_USER
    not_accepting_task_reason: int = 0


@dataclass
class RunningTask:
    """yadcc/api/scheduler.proto:233-238."""

    servant_task_id: int = 0
    task_grant_id: int = 0
    servant_location: str = ""
    task_digest: str = ""


class StateError(RuntimeError):
    """yd_import_state refused an export; `code` is one of _abi.STATE_* (ydstate.h)."""

    NAMES = {1: "malformed export", 2: "the handle is not fresh", 3: "the export's config differs from the handle's",
             4: "range-sharded handles have no state export",
             5: "the export's lease window does not fit the device's free memory now"}

    def __init__(self, code: int):
        super().__init__(f"yd_import_state: {self.NAMES.get(code, code)}")
        self.code = code


def _ns(seconds: float | int) -> int:
    return int(round(seconds * 1_000_000_000))


def pack_requests(reqs: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
    """REQ_DTYPE -> REQ16_DTYPE (yd_task_req16).  Leases must be whole milliseconds below 2^31 ms -- the RPC
    surface's unit (scheduler.proto next_keep_alive_in_ms)."""
    ns = reqs["expires_in_ns"]
    assert (ns % 1_000_000 == 0).all() and (ns >= 0).all() and (ns < (1 << 31) * 1_000_000).all()
    if out is None:
        out = np.empty(reqs.shape[0], dtype=_abi.REQ16_DTYPE)
    out["env_id"] = reqs["env_id"]
    out["min_version"] = reqs["min_version"]
    out["requestor_ip"] = reqs["requestor_ip"]
    out["lease"] = (ns // 1_000_000).astype(np.uint32) | np.where(
        reqs["flags"] & _abi.REQ_FLAG_PREFETCH, np.uint32(_abi.LEASE_PREFETCH), np.uint32(0))
    return out


def unpack_grants(g8: np.ndarray, ids) -> np.ndarray:
    """GRANT8 + PACKED_IDS -> GRANT_DTYPE (yd_unpack_grant)."""
    out = np.zeros(g8.shape[0], dtype=GRANT_DTYPE)
    so = g8["status_ordinal"]
    out["status"] = so >> 30
    out["servant_index"] = g8["servant_index"]
    granted = out["status"] == _abi.STATUS_GRANTED
    out["task_id"] = np.where(
        granted, np.uint64(ids["first_task_id"]) + (so & 0x3FFFFFFF).astype(np.uint64) * np.uint64(ids["stride"]), np.uint64(0))
    return out


class TaskDispatcher:
    def __init__(
        self,
        library=None,
        *,
        device: int = 0,
        servant_min_memory_for_accepting_new_task: str | None = None,
        solver: int = 0,
        graphs: bool = True,
        merge_self: bool = True,
        tiny: bool = True,
        fused: bool = True,
        id_stride: int = 0,
        id_offset: int = 0,
    ):
        self._lib = library if isinstance(library, C.CDLL) else _abi.load_library(library)
        cfg = _abi.yd_config(
            abi_version=_abi.ABI_VERSION,
            device=device,
            servant_min_memory_for_accepting_new_task=(
                servant_min_memory_for_accepting_new_task.encode()
                if servant_min_memory_for_accepting_new_task is not None
                else None
            ),
            solver=solver,
            # bit 0: do not capture the solve into a CUDA graph (per-phase timing); bit 1 (test switch): components
            # whose requestors are servants go to the sequential solver instead of the merge solver
            # bit 2 (test switch): batches of <= 8 requests take the full pipeline instead of the one-launch path
            # bit 3 (test switch): no fused front kernel (fused.cuh) -- the kernel-by-kernel pipeline at every size
            reserved=(0 if graphs else 1) | (0 if merge_self else 2) | (0 if tiny else 4) | (0 if fused else 8),
            id_stride=id_stride,
            id_offset=id_offset,
        )
        self._h = self._lib.yd_create(C.byref(cfg))
        if not self._h:
            raise RuntimeError(
                f"yd_create failed for backend {self.backend!r} ({self._lib._yd_path}); "
                "the CUDA backend needs an sm_90 GPU (H100) and never falls back to the CPU"
            )
        self._env_ids: dict[str, int] = {}
        self._ip_ids: dict[str, int] = {}

    # -- lifecycle ---------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.yd_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def backend(self) -> str:
        return self._lib.yd_backend_name().decode()

    # -- interning ---------------------------------------------------------
    def intern_env(self, compiler_digest: str) -> int:
        v = self._env_ids.get(compiler_digest)
        if v is None:
            b = compiler_digest.encode()
            v = self._env_ids[compiler_digest] = self._lib.yd_intern_env(self._h, b, len(b))
        return v

    def intern_ip(self, requestor_ip: str) -> int:
        v = self._ip_ids.get(requestor_ip)
        if v is None:
            b = requestor_ip.encode()
            v = self._ip_ids[requestor_ip] = self._lib.yd_intern_ip(self._h, b, len(b))
        return v

    # -- task servant allocation (task_dispatcher.h:126-155) ----------------
    def wait_for_starting_new_tasks(
        self, reqs: np.ndarray, now: float = 0.0, *, now_ns: int | None = None, out: np.ndarray | None = None
    ) -> np.ndarray:
        """n sequential WaitForStartingNewTask calls (cc:93-140); THE hot path.

        `reqs` is a REQ_DTYPE array (ideally in memory from `alloc_requests`);
        returns a GRANT_DTYPE array.
        """
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        n = reqs.shape[0]
        if out is None:
            out = np.empty(n, dtype=GRANT_DTYPE)
        assert out.dtype == GRANT_DTYPE and out.shape[0] >= n and out.flags.c_contiguous
        self._lib.yd_wait_for_starting_new_tasks(
            self._h, now_ns if now_ns is not None else _ns(now), reqs.ctypes.data, n, out.ctypes.data
        )
        return out[:n]

    def wait_for_starting_new_tasks_packed(
        self, reqs16: np.ndarray, now: float = 0.0, *, now_ns: int | None = None, out8: np.ndarray | None = None,
        unpack: bool = True,
    ) -> np.ndarray | tuple[np.ndarray, np.ndarray]:
        """The same decisions through the packed interface (yd_wait_for_starting_new_tasks_packed): 16-byte
        requests (`pack_requests`), 8-byte grants.  unpack=True returns a GRANT_DTYPE array like
        wait_for_starting_new_tasks; unpack=False returns (GRANT8 array, PACKED_IDS record)."""
        assert reqs16.dtype == _abi.REQ16_DTYPE and reqs16.flags.c_contiguous
        n = reqs16.shape[0]
        if out8 is None:
            out8 = np.empty(n, dtype=_abi.GRANT8_DTYPE)
        assert out8.dtype == _abi.GRANT8_DTYPE and out8.shape[0] >= n and out8.flags.c_contiguous
        ids = np.zeros(1, dtype=_abi.PACKED_IDS_DTYPE)
        self._lib.yd_wait_for_starting_new_tasks_packed(
            self._h, now_ns if now_ns is not None else _ns(now), reqs16.ctypes.data, n, out8.ctypes.data, ids.ctypes.data
        )
        if not unpack:
            return out8[:n], ids[0]
        return unpack_grants(out8[:n], ids[0])

    def make_requests(
        self,
        n: int,
        compiler_digest: str | Sequence[str],
        requestor_ip: str | Sequence[str],
        min_version: int | Sequence[int] = 0,
        expires_in: float = 15.0,
        prefetching: bool = False,
        pinned: bool = False,
    ) -> np.ndarray:
        r = self.alloc_requests(n) if pinned else np.zeros(n, dtype=REQ_DTYPE)
        if isinstance(compiler_digest, str):
            r["env_id"] = self.intern_env(compiler_digest)
        else:
            r["env_id"] = [self.intern_env(d) for d in compiler_digest]
        if isinstance(requestor_ip, str):
            r["requestor_ip"] = self.intern_ip(requestor_ip)
        else:
            r["requestor_ip"] = [self.intern_ip(d) for d in requestor_ip]
        r["min_version"] = min_version
        r["flags"] = _abi.REQ_FLAG_PREFETCH if prefetching else 0
        r["expires_in_ns"] = _ns(expires_in)
        return r

    def wait_for_starting_new_task(
        self,
        requestor_ip: str,
        min_version: int,
        compiler_digest: str,
        expires_in: float,
        timeout: float | None = None,
        prefetching: bool = False,
        *,
        now: float = 0.0,
    ) -> TaskAllocation | WaitStatus:
        """One decision; returns a TaskAllocation or the WaitStatus error."""
        del timeout  # zero-wait discipline
        r = self.make_requests(1, compiler_digest, requestor_ip, min_version, expires_in, prefetching)
        g = self.wait_for_starting_new_tasks(r, now)[0]
        if g["status"] == _abi.STATUS_GRANTED:
            return TaskAllocation(int(g["task_id"]), self.servant_location(int(g["servant_index"])))
        return WaitStatus(int(g["status"]))

    def stage_requests(self, reqs: np.ndarray) -> None:
        """Copy the pending queue into HBM ahead of the solve (yd_stage_requests)."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        self._lib.yd_stage_requests(self._h, reqs.ctypes.data, reqs.shape[0])

    def wait_for_staged_tasks(self, n: int, now: float = 0.0, out: np.ndarray | None = None) -> np.ndarray:
        """Decide the first n staged requests (queue already resident in HBM)."""
        if out is None:
            out = np.zeros(n, dtype=GRANT_DTYPE)
        assert out.dtype == GRANT_DTYPE and out.flags.c_contiguous and out.shape[0] >= n
        self._lib.yd_wait_for_staged_tasks(self._h, _ns(now), n, out.ctypes.data)
        return out[:n]

    def wait_for_starting_task_rpcs(self, rpcs: np.ndarray, now: float = 0.0):
        """A batch of SchedulerServiceImpl::WaitForStartingTask bodies
        (scheduler_service_impl.cc:209-271): returns (results, grants) where
        results[i] = (status, n_grants, first_grant) and grants is a GRANT_DTYPE array."""
        assert rpcs.dtype == _abi.RPC_WAIT_DTYPE and rpcs.flags.c_contiguous
        n = rpcs.shape[0]
        cap = int(self._lib.yd_rpc_expanded_requests(self._h, rpcs.ctypes.data, n))  # counts clamped to what can be granted
        results = np.zeros(n, dtype=_abi.RPC_RESULT_DTYPE)
        grants = np.zeros(max(cap, 1), dtype=GRANT_DTYPE)
        k = self._lib.yd_wait_for_starting_task_rpcs(self._h, _ns(now), rpcs.ctypes.data, n, results.ctypes.data,
                                                     grants.ctypes.data, cap)
        if k == (1 << 64) - 1:
            raise ValueError("grant buffer too small")
        return results, grants[:k]

    def keep_task_alive(self, task_id: int, new_expires_in: float, *, now: float = 0.0) -> bool:
        return bool(self.keep_tasks_alive([task_id], new_expires_in, now=now)[0])

    def keep_tasks_alive(self, task_ids: Iterable[int], new_expires_in: float, *, now: float = 0.0) -> np.ndarray:
        ids = np.ascontiguousarray(np.asarray(list(task_ids) if not isinstance(task_ids, np.ndarray) else task_ids, dtype=np.uint64))
        ok = np.zeros(ids.shape[0], dtype=np.uint8)
        self._lib.yd_keep_task_alive(self._h, _ns(now), ids.ctypes.data, ids.shape[0], _ns(new_expires_in), ok.ctypes.data)
        return ok.astype(bool)

    def free_task(self, task_id: int) -> None:
        self.free_tasks([task_id])

    def free_tasks(self, task_ids: Iterable[int]) -> None:
        ids = np.ascontiguousarray(np.asarray(list(task_ids) if not isinstance(task_ids, np.ndarray) else task_ids, dtype=np.uint64))
        self._lib.yd_free_tasks(self._h, ids.ctypes.data, ids.shape[0])

    # -- servant maintenance (task_dispatcher.h:157-181) -------------------
    def _servant_struct(self, servant: Servant, keep: list) -> "_abi.yd_servant":
        envs = [e.encode() for e in servant.environments]
        arr = (C.c_char_p * max(len(envs), 1))(*envs)
        rep = servant.reported_location if servant.reported_location is not None else servant.observed_location
        keep.append((envs, arr))
        return _abi.yd_servant(
            version=servant.version,
            priority=servant.priority,
            not_accepting_task_reason=servant.not_accepting_task_reason,
            num_envs=len(envs),
            observed_location=servant.observed_location.encode(),
            reported_location=rep.encode(),
            env_digests=arr,
            num_processors=servant.num_processors,
            current_load=servant.current_load,
            max_tasks=servant.max_tasks,
            total_memory_in_bytes=servant.total_memory_in_bytes,
            memory_available_in_bytes=servant.memory_available_in_bytes,
        )

    def keep_servant_alive(self, servant: Servant, expires_in: float, *, now: float = 0.0) -> None:
        keep: list = []
        sv = self._servant_struct(servant, keep)
        self._lib.yd_keep_servant_alive(self._h, _ns(now), C.byref(sv), _ns(expires_in))

    def keep_servants_alive(self, servants: Sequence[Servant], expires_in: Sequence[float] | float, *, now: float = 0.0) -> None:
        """KeepServantAlive for a whole tick's heartbeats in one call (yd_keep_servants_alive)."""
        n = len(servants)
        keep: list = []
        structs = [self._servant_struct(sv, keep) for sv in servants]  # (they own the byte strings the array points to)
        arr = (_abi.yd_servant * max(n, 1))(*structs)
        exp = [expires_in] * n if isinstance(expires_in, (int, float)) else list(expires_in)
        ex = (C.c_int64 * max(n, 1))(*[_ns(e) for e in exp])
        self._lib.yd_keep_servants_alive(self._h, _ns(now), arr, ex, n)
        del structs, keep

    def notify_servants_running_tasks(self, batch: Sequence[tuple[str, Sequence[RunningTask]]]) -> list[list[int]]:
        """NotifyServantRunningTasks for many servants in one call: [(location, tasks)] -> unknown ids per item."""
        n = len(batch)
        items = (_abi.yd_heartbeat_item * max(n, 1))()
        keep = []
        total = 0
        for i, (loc, tasks) in enumerate(batch):
            m = len(tasks)
            arr = (_abi.yd_running_task * max(m, 1))()
            for k, t in enumerate(tasks):
                l2, dig = t.servant_location.encode(), t.task_digest.encode()
                keep.append((l2, dig))
                arr[k] = _abi.yd_running_task(t.servant_task_id, t.task_grant_id, l2, dig)
            lb = loc.encode()
            keep.append((arr, lb))
            items[i] = _abi.yd_heartbeat_item(lb, arr, m)
            total += m
        out = (C.c_uint64 * max(total, 1))()
        counts = (C.c_size_t * max(n, 1))()
        self._lib.yd_notify_servants_running_tasks(self._h, items, n, out, counts)
        res, at = [], 0
        for i in range(n):
            res.append([int(out[at + k]) for k in range(counts[i])])
            at += counts[i]
        return res

    def notify_servant_running_tasks(self, servant_location: str, tasks: Sequence[RunningTask]) -> list[int]:
        n = len(tasks)
        arr = (_abi.yd_running_task * max(n, 1))()
        keep = []
        for i, t in enumerate(tasks):
            loc, dig = t.servant_location.encode(), t.task_digest.encode()
            keep.append((loc, dig))
            arr[i] = _abi.yd_running_task(t.servant_task_id, t.task_grant_id, loc, dig)
        out = (C.c_uint64 * max(n, 1))()
        k = self._lib.yd_notify_servant_running_tasks(self._h, servant_location.encode(), arr, n, out)
        return [int(out[i]) for i in range(k)]

    def get_running_tasks(self) -> list[RunningTask]:
        n = self._lib.yd_get_running_tasks(self._h, None, 0)
        arr = (_abi.yd_running_task * max(n, 1))()
        n = min(n, self._lib.yd_get_running_tasks(self._h, arr, n))
        return [
            RunningTask(
                int(arr[i].servant_task_id),
                int(arr[i].task_grant_id),
                (arr[i].servant_location or b"").decode(),
                (arr[i].task_digest or b"").decode(),
            )
            for i in range(n)
        ]

    def on_expiration_timer(self, *, now: float) -> None:
        self._lib.yd_on_expiration_timer(self._h, _ns(now))

    # -- compilation-cache bloom pre-filter (flare SaltedBloomFilter) ------------
    @staticmethod
    def _key_matrix(keys) -> np.ndarray:
        """Fixed-length keys as an (n, key_len) uint8 matrix."""
        if isinstance(keys, np.ndarray) and keys.dtype == np.uint8 and keys.ndim == 2:
            return np.ascontiguousarray(keys)
        b = [k.encode() if isinstance(k, str) else bytes(k) for k in keys]
        n = len(b)
        ln = len(b[0]) if n else 0
        assert all(len(x) == ln for x in b), "keys of one call must have the same length"
        return np.frombuffer(b"".join(b), dtype=np.uint8).reshape(n, ln).copy()

    def bloom_reset(self, size_in_bits: int = 27584639, num_hashes: int = 10) -> None:
        """Defaults: yadcc/cache/bloom_filter_generator.h:65-68."""
        if self._lib.yd_bloom_reset(self._h, size_in_bits, num_hashes) != 0:
            raise ValueError("bad bloom filter geometry")

    def bloom_load(self, data: bytes, num_hashes: int = 10) -> None:
        buf = np.frombuffer(data, dtype=np.uint8)
        if self._lib.yd_bloom_load(self._h, buf.ctypes.data, len(buf), num_hashes) != 0:
            raise ValueError("bloom filter size must be a power of two")

    def bloom_add(self, keys) -> None:
        m = self._key_matrix(keys)
        if len(m):
            self._lib.yd_bloom_add(self._h, m.ctypes.data, m.shape[0], m.shape[1], m.strides[0])

    def bloom_possibly_contains(self, keys) -> np.ndarray:
        m = self._key_matrix(keys)
        out = np.zeros(m.shape[0], dtype=np.uint8)
        if len(m):
            self._lib.yd_bloom_possibly_contains(self._h, m.ctypes.data, m.shape[0], m.shape[1], m.strides[0],
                                                 out.ctypes.data)
        return out.astype(bool)

    def bloom_bytes(self) -> bytes:
        n = self._lib.yd_bloom_get_bytes(self._h, None, 0)
        out = np.zeros(n, dtype=np.uint8)
        self._lib.yd_bloom_get_bytes(self._h, out.ctypes.data, n)
        return out.tobytes()

    # -- in-flight task index (RunningTaskKeeper, running_task_keeper.cc:40-75) ----
    def running_index_refresh(self) -> int:
        """Refresh(): rebuild digest -> running task from the current bookkeeping.
        Returns the snapshot length."""
        return int(self._lib.yd_running_index_refresh(self._h))

    def running_index_size(self) -> int:
        return int(self._lib.yd_running_index_size(self._h))

    def find_running_tasks(self, digests) -> np.ndarray:
        """TryFindTask for a whole queue of (equal-length) task digests.  Returns a
        RUNNING_HIT array: found, snapshot_index, servant_task_id."""
        m = self._key_matrix(digests)
        out = np.zeros(m.shape[0], dtype=_abi.RUNNING_HIT_DTYPE)
        if len(m):
            self._lib.yd_running_index_find(self._h, m.ctypes.data, m.shape[0], m.shape[1], m.strides[0],
                                            out.ctypes.data)
        return out

    def filter_and_wait_for_starting_new_tasks(self, reqs: np.ndarray, cache_keys=None, task_digests=None, now: float = 0.0,
                                               out: np.ndarray | None = None, verdict_out: np.ndarray | None = None,
                                               want_hits: bool = True):
        """BASELINE configs[3] in one call (yd_filter_and_wait_for_starting_new_tasks): bloom pre-filter on the
        cache keys, in-flight dedupe on the task digests, then the solve over what is left.  Returns
        (verdicts uint8[n], hits RUNNING_HIT[n], grants GRANT[n_offered])."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        n = reqs.shape[0]
        f = _abi.yd_prefilter()
        km = dm = None
        if cache_keys is not None:
            km = self._key_matrix(cache_keys)
            assert km.shape[0] >= n
            f.cache_keys, f.cache_key_len, f.cache_key_stride = km.ctypes.data, km.shape[1], km.strides[0]
        if task_digests is not None:
            dm = self._key_matrix(task_digests)
            assert dm.shape[0] >= n
            f.task_digests, f.task_digest_len, f.task_digest_stride = dm.ctypes.data, dm.shape[1], dm.strides[0]
        verdict = verdict_out[:n] if verdict_out is not None else np.zeros(n, dtype=np.uint8)
        assert verdict.dtype == np.uint8 and verdict.shape[0] == n and verdict.flags.c_contiguous
        hits = np.zeros(n, dtype=_abi.RUNNING_HIT_DTYPE) if want_hits else None
        if out is None:
            out = np.zeros(max(n, 1), dtype=GRANT_DTYPE)
        assert out.dtype == GRANT_DTYPE and out.shape[0] >= n and out.flags.c_contiguous
        k = self._lib.yd_filter_and_wait_for_starting_new_tasks(self._h, _ns(now), reqs.ctypes.data, n, C.byref(f),
                                                                verdict.ctypes.data, hits.ctypes.data if want_hits else None,
                                                                out.ctypes.data)
        return verdict, hits, out[: int(k)]

    def running_index_entry(self, snapshot_index: int) -> RunningTask | None:
        t = _abi.yd_running_task()
        import ctypes as C

        if not self._lib.yd_running_index_entry(self._h, int(snapshot_index), C.byref(t)):
            return None
        return RunningTask(int(t.servant_task_id), int(t.task_grant_id), (t.servant_location or b"").decode(),
                           (t.task_digest or b"").decode())

    # -- state export / import (include/ydstate.h) --------------------------
    def _state_fn(self, name: str):
        fn = getattr(self._lib, name, None)
        if fn is None:
            raise NotImplementedError(f"{self._lib._yd_path} does not export {name}")
        return fn

    def export_state(self, now: float = 0.0, *, now_ns: int | None = None) -> bytes:
        """The handle's decision state (servants, leases, next task id, running-task bookkeeping, intern
        tables) in the versioned format of ydstate.h, times relative to `now`."""
        fn = self._state_fn("yd_export_state")
        t = now_ns if now_ns is not None else _ns(now)
        n = fn(self._h, t, None, 0)
        if n == 0:
            raise StateError(_abi.STATE_UNSUPPORTED)
        buf = C.create_string_buffer(n)
        m = fn(self._h, t, buf, n)
        assert m == n, (m, n)
        return buf.raw

    def import_state(self, blob: bytes, now: float = 0.0, *, now_ns: int | None = None) -> None:
        """Load an export into this handle, which must be fresh (no call since construction).  Times are
        rebased onto `now`.  Raises StateError with the ydstate.h status code if the export is refused."""
        fn = self._state_fn("yd_import_state")
        data = bytes(blob)
        rc = fn(self._h, now_ns if now_ns is not None else _ns(now), data, len(data))
        if rc != _abi.STATE_OK:
            raise StateError(rc)

    # -- introspection -----------------------------------------------------
    def num_servants(self) -> int:
        return int(self._lib.yd_num_servants(self._h))

    def servant_personality(self, index: int) -> Servant | None:
        """ServantPersonality of registry position `index` as last reported."""
        sv = _abi.yd_servant()
        if not self._lib.yd_get_servant_personality(self._h, int(index), C.byref(sv)):
            return None
        return Servant(
            observed_location=(sv.observed_location or b"").decode(),
            reported_location=(sv.reported_location or b"").decode(),
            environments=[sv.env_digests[i].decode() for i in range(sv.num_envs)],
            version=sv.version, num_processors=sv.num_processors, current_load=sv.current_load,
            total_memory_in_bytes=sv.total_memory_in_bytes, memory_available_in_bytes=sv.memory_available_in_bytes,
            max_tasks=sv.max_tasks, priority=sv.priority, not_accepting_task_reason=sv.not_accepting_task_reason)

    def servant_location(self, index: int) -> str | None:
        v = self._lib.yd_servant_location(self._h, index)
        return v.decode() if v is not None else None

    def servant_state(self) -> np.ndarray:
        n = self.num_servants()
        out = np.zeros(n, dtype=SERVANT_STATE_DTYPE)
        self._lib.yd_get_servant_state(self._h, out.ctypes.data, n)
        return out

    def next_task_id(self) -> int:
        return int(self._lib.yd_next_task_id(self._h))

    def num_tasks(self) -> int:
        return int(self._lib.yd_num_tasks(self._h))

    def dump_internals(self) -> dict:
        n = self._lib.yd_dump_internals_json(self._h, None, 0)
        buf = C.create_string_buffer(n + 1)
        self._lib.yd_dump_internals_json(self._h, buf, len(buf))
        return json.loads(buf.value.decode())

    def last_solve_stats(self) -> dict | None:
        st = _abi.yd_solve_stats()
        if not self._lib.yd_last_solve_stats(self._h, C.byref(st)):
            return None
        return {k: getattr(st, k) for k, _ in st._fields_}

    def parse_size(self, text: str) -> int | None:
        v = C.c_uint64()
        return int(v.value) if self._lib.yd_parse_size(text.encode(), C.byref(v)) else None

    # -- pinned staging ----------------------------------------------------
    def _alloc(self, n: int, dtype: np.dtype) -> np.ndarray:
        nbytes = max(n, 1) * dtype.itemsize
        p = self._lib.yd_alloc_host(nbytes)
        if not p:
            raise MemoryError("yd_alloc_host failed")
        buf = (C.c_char * nbytes).from_address(p)
        arr = np.frombuffer(buf, dtype=dtype, count=n)
        lib = self._lib
        # keep the allocation alive as long as the array; free it afterwards
        import weakref

        weakref.finalize(buf, lib.yd_free_host, p)
        arr[...] = np.zeros((), dtype=dtype)
        return arr

    def alloc_requests(self, n: int) -> np.ndarray:
        return self._alloc(n, REQ_DTYPE)

    def alloc_grants(self, n: int) -> np.ndarray:
        return self._alloc(n, GRANT_DTYPE)

    def alloc_requests16(self, n: int) -> np.ndarray:
        return self._alloc(n, _abi.REQ16_DTYPE)

    def alloc_grants8(self, n: int) -> np.ndarray:
        return self._alloc(n, _abi.GRANT8_DTYPE)
