"""SchedulerServiceImpl's handlers over the C ABI (include/ydservice.h): the mirror of
yadcc/scheduler/scheduler_service_impl.cc:67-333 a front end (or a test) talks to."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np

from . import _abi
from ._abi import GRANT_DTYPE
from .dispatcher import RunningTask, TaskDispatcher, _ns

STATUS_OK = 0
STATUS_NO_QUOTA_AVAILABLE = 1001
STATUS_ACCESS_DENIED = 1003
STATUS_INVALID_ARGUMENT = 1004
STATUS_VERSION_TOO_OLD = 1005
STATUS_ENVIRONMENT_NOT_AVAILABLE = 1006
REASON_BEHIND_NAT = 4
REASON_NOT_VERIFIED = 100


@dataclass
class HeartbeatRequest:
    """yadcc/api/scheduler.proto:63-118 plus the peer address the RPC layer observed."""

    token: str = ""
    location: str = ""
    remote_ip: str = ""
    remote_is_ipv6: bool = False
    next_heartbeat_in_ms: int = 1000
    version: int = 0
    num_processors: int = 0
    current_load: int = 0
    servant_priority: int = 0
    not_accepting_task_reason: int = 0
    capacity: int = 0
    total_memory_in_bytes: int = 0
    memory_available_in_bytes: int = 0
    env_digests: Sequence[str] = field(default_factory=list)
    running_tasks: Sequence[RunningTask] = field(default_factory=list)


@dataclass
class HeartbeatResponse:
    status: int
    acceptable_tokens: list[str]
    expired_tasks: list[int]


class SchedulerService:
    def __init__(self, dispatcher: TaskDispatcher, *, acceptable_user_tokens: str, acceptable_servant_tokens: str,
                 min_daemon_version: int = 0, serving_daemon_token_rollout_interval: int = 3600, token_seed: int = 0,
                 now: float = 0.0):
        """`dispatcher` may also be a RangeShardedDispatcher: the service then answers for the whole group
        (yd_shard_service_create).  Building it is collective, and every rank's service must be fed the same calls;
        every rank then gives the same answers and hands out rank 0's serving-daemon tokens."""
        group = None
        if not isinstance(dispatcher, TaskDispatcher):  # a RangeShardedDispatcher
            group, dispatcher = dispatcher, dispatcher.local
        self.group = group
        self.dispatcher = dispatcher
        self._lib = dispatcher._lib
        create = self._lib.yd_service_create
        if group is not None and group.native:
            create = self._lib.yd_shard_service_create
        elif group is not None and token_seed == 0 and group.world > 1:
            # replicas over gloo: the same tokens on every rank from a seed rank 0 draws
            import secrets

            import torch.distributed as dist

            seeds: list = [None] * group.world
            dist.all_gather_object(seeds, secrets.randbits(64) or 1, group=group.group)
            token_seed = seeds[0]
        cfg = _abi.yd_service_config(acceptable_user_tokens.encode(), acceptable_servant_tokens.encode(),
                                     min_daemon_version, serving_daemon_token_rollout_interval, token_seed)
        self._h = create(dispatcher._h, _ns(now), C.byref(cfg))
        if not self._h:
            raise ValueError("both token lists must be non-empty (token_verifier.cc:58-59)")

    def close(self):
        if self._h:
            self._lib.yd_service_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _heartbeat_struct(req: HeartbeatRequest, keep: list):
        """The request struct and the response's expired-ids buffer; `keep` owns what they point to."""
        envs = [e.encode() for e in req.env_digests]
        env_arr = (C.c_char_p * max(len(envs), 1))(*envs)
        n = len(req.running_tasks)
        tasks = (_abi.yd_running_task * max(n, 1))()
        for i, t in enumerate(req.running_tasks):
            loc, dig = t.servant_location.encode(), t.task_digest.encode()
            keep.append((loc, dig))
            tasks[i] = _abi.yd_running_task(t.servant_task_id, t.task_grant_id, loc, dig)
        expired = (C.c_uint64 * max(n, 1))()
        strs = (req.token.encode(), req.location.encode(), req.remote_ip.encode())
        keep.append((envs, env_arr, tasks, expired, strs))
        r = _abi.yd_heartbeat_request(
            strs[0], strs[1], strs[2], int(req.remote_is_ipv6),
            req.next_heartbeat_in_ms, req.version, req.num_processors, req.current_load, req.servant_priority,
            req.not_accepting_task_reason, req.capacity, len(envs), req.total_memory_in_bytes,
            req.memory_available_in_bytes, env_arr, tasks, n)
        return r, expired

    @staticmethod
    def _heartbeat_answer(st: int, resp, expired) -> HeartbeatResponse:
        if st != STATUS_OK:
            return HeartbeatResponse(st, [], [])
        return HeartbeatResponse(st, [resp.acceptable_tokens[i].decode() for i in range(3)],
                                 [int(expired[i]) for i in range(resp.n_expired_tasks)])

    def heartbeat(self, req: HeartbeatRequest, *, now: float = 0.0) -> HeartbeatResponse:
        keep: list = []
        r, expired = self._heartbeat_struct(req, keep)
        resp = _abi.yd_heartbeat_response()
        resp.expired_tasks = expired
        st = self._lib.yd_service_heartbeat(self._h, _ns(now), C.byref(r), C.byref(resp))
        return self._heartbeat_answer(st, resp, expired)

    def heartbeats(self, reqs: Sequence[HeartbeatRequest], *, now: float = 0.0) -> list[HeartbeatResponse]:
        """A run of Heartbeat RPCs in one call (yd_service_heartbeats): the answers of `heartbeat` on each in order."""
        n = len(reqs)
        keep: list = []
        rq = (_abi.yd_heartbeat_request * max(n, 1))()
        rs = (_abi.yd_heartbeat_response * max(n, 1))()
        bufs = []
        for i, req in enumerate(reqs):
            rq[i], expired = self._heartbeat_struct(req, keep)
            rs[i].expired_tasks = expired
            bufs.append(expired)
        st = (C.c_int * max(n, 1))()
        self._lib.yd_service_heartbeats(self._h, _ns(now), rq, n, rs, st)
        return [self._heartbeat_answer(st[i], rs[i], bufs[i]) for i in range(n)]

    def get_config(self, token: str, *, now: float = 0.0) -> tuple[int, str | None]:
        out = C.c_char_p()
        st = self._lib.yd_service_get_config(self._h, _ns(now), token.encode(), C.byref(out))
        return st, (out.value.decode() if st == STATUS_OK else None)

    def wait_for_starting_tasks(self, tokens: Sequence[str], rpcs: np.ndarray, *, now: float = 0.0):
        """Batch of WaitForStartingTask RPCs: returns (results, grants) like
        TaskDispatcher.wait_for_starting_task_rpcs, with ACCESS_DENIED for bad tokens."""
        assert rpcs.dtype == _abi.RPC_WAIT_DTYPE and rpcs.flags.c_contiguous and len(tokens) == len(rpcs)
        n = rpcs.shape[0]
        tok = (C.c_char_p * max(n, 1))(*[t.encode() for t in tokens])
        cap = int(self._lib.yd_rpc_expanded_requests(self.dispatcher._h, rpcs.ctypes.data, n))
        results = np.zeros(n, dtype=_abi.RPC_RESULT_DTYPE)
        grants = np.zeros(max(cap, 1), dtype=GRANT_DTYPE)
        k = self._lib.yd_service_wait_for_starting_tasks(self._h, _ns(now), tok, rpcs.ctypes.data, n,
                                                         results.ctypes.data, grants.ctypes.data, cap)
        return results, grants[:k]

    def keep_task_alive(self, token: str, task_grant_ids, next_keep_alive_in_ms: int, *, now: float = 0.0):
        ids = np.ascontiguousarray(np.asarray(task_grant_ids, dtype=np.uint64))
        ok = np.zeros(len(ids), dtype=np.uint8)
        st = self._lib.yd_service_keep_task_alive(self._h, _ns(now), token.encode(), next_keep_alive_in_ms,
                                                  ids.ctypes.data, len(ids), ok.ctypes.data)
        return st, ok.astype(bool)

    def free_task(self, token: str, task_grant_ids) -> int:
        ids = np.ascontiguousarray(np.asarray(task_grant_ids, dtype=np.uint64))
        return self._lib.yd_service_free_task(self._h, token.encode(), ids.ctypes.data, len(ids))

    def keep_tasks_alive(self, requests, *, now: float = 0.0) -> list[tuple[int, np.ndarray]]:
        """A run of KeepTaskAlive RPCs, [(token, task_grant_ids, next_keep_alive_in_ms)], in one call
        (yd_service_keep_tasks_alive): the answers of `keep_task_alive` on each in order."""
        n = len(requests)
        rq = (_abi.yd_keep_task_alive_request * max(n, 1))()
        keep = []
        for i, (token, task_grant_ids, ms) in enumerate(requests):
            ids = np.ascontiguousarray(np.asarray(task_grant_ids, dtype=np.uint64))
            ok = np.zeros(max(len(ids), 1), dtype=np.uint8)
            tok = token.encode()
            keep.append((ids, ok, tok))
            rq[i] = _abi.yd_keep_task_alive_request(tok, ms, ids.ctypes.data, len(ids), ok.ctypes.data)
        st = (C.c_int * max(n, 1))()
        self._lib.yd_service_keep_tasks_alive(self._h, _ns(now), rq, n, st)
        return [(st[i], keep[i][1][:len(keep[i][0])].astype(bool)) for i in range(n)]

    def free_tasks(self, requests) -> list[int]:
        """A run of FreeTask RPCs, [(token, task_grant_ids)], in one call (yd_service_free_tasks): the statuses of
        `free_task` on each in order."""
        n = len(requests)
        rq = (_abi.yd_free_task_request * max(n, 1))()
        keep = []
        for i, (token, task_grant_ids) in enumerate(requests):
            ids = np.ascontiguousarray(np.asarray(task_grant_ids, dtype=np.uint64))
            tok = token.encode()
            keep.append((ids, tok))
            rq[i] = _abi.yd_free_task_request(tok, ids.ctypes.data, len(ids))
        st = (C.c_int * max(n, 1))()
        self._lib.yd_service_free_tasks(self._h, rq, n, st)
        return [st[i] for i in range(n)]

    def get_running_tasks(self) -> list[RunningTask]:
        n = self._lib.yd_service_get_running_tasks(self._h, None, 0)
        arr = (_abi.yd_running_task * max(n, 1))()
        n = min(n, self._lib.yd_service_get_running_tasks(self._h, arr, n))
        return [RunningTask(int(arr[i].servant_task_id), int(arr[i].task_grant_id),
                            (arr[i].servant_location or b"").decode(), (arr[i].task_digest or b"").decode())
                for i in range(n)]

    # -- FlareStd wire front end (include/ydwire.h) ---------------------------------
    def handle_frames(self, frames, *, now: float = 0.0, out_cap: int | None = None):
        """frames: [(bytes, remote_ip[, is_ipv6])], the first frame of each is handled, in order
        (consecutive Heartbeat, WaitForStartingTask, KeepTaskAlive or FreeTask frames as one batch).  Returns a list of
        (verdict, consumed, status, response_bytes)."""
        n = len(frames)
        ins = (_abi.yd_wire_in * max(n, 1))()
        keep = []
        for i, f in enumerate(frames):
            data, ip = f[0], f[1]
            buf = C.create_string_buffer(bytes(data), len(data))
            ipb = ip.encode()
            keep.append((buf, ipb))
            ins[i] = _abi.yd_wire_in(C.cast(buf, C.c_void_p), len(data), ipb, int(f[2]) if len(f) > 2 else 0, 0)
        cap = out_cap if out_cap is not None else 65536 * max(n, 1)
        out = C.create_string_buffer(cap)
        outs = (_abi.yd_wire_out * max(n, 1))()
        total = self._lib.yd_wire_handle_frames(self._h, _ns(now), ins, n, C.cast(out, C.c_void_p), cap, outs)
        if total == (1 << 64) - 1:
            raise ValueError("response buffer too small")
        return [(outs[i].verdict, outs[i].consumed, outs[i].status, out.raw[outs[i].offset:outs[i].offset + outs[i].len])
                for i in range(n)]

    def call(self, method: str, body: bytes, remote_ip: str, *, now: float = 0.0, remote_is_ipv6: bool = False):
        """One call at message-body level (yd_wire_call): returns (status, description, response bytes)."""
        cap = 1 << 20
        out = C.create_string_buffer(cap)
        n = C.c_size_t(0)
        desc = C.c_char_p()
        st = self._lib.yd_wire_call(self._h, _ns(now), method.encode(), remote_ip.encode(), int(remote_is_ipv6), body,
                                    len(body), C.cast(out, C.c_void_p), cap, C.byref(n), C.byref(desc))
        return st, (desc.value or b"").decode(), out.raw[:n.value]
