"""One logical scheduler over several GPUs (SURVEY.md 8(e), option 1).

Decisions couple only through per-servant `running_tasks`, so servants that share no
compiler digest never interact: the connected components of the digest<->servant graph
are independent FIFO sub-queues (the sharding the reference's authors propose at
yadcc/scheduler/task_dispatcher.h:286-288).  `ShardedDispatcher` gives every rank a
subset of the components -- their servants, their digests and the requests for them --
and one process per GPU runs an ordinary `TaskDispatcher` on its share.  No servant
state ever crosses ranks.

The only thing the shards share is the task-id space.  Two modes:

* "strided" (default): the library itself hands out id = local_id * world + rank
  (`yd_config.id_stride / id_offset`) and ignores ids that are not its own -- no
  communication at all.  Task-grant ids are opaque lease tokens on the wire
  (scheduler.proto:181-238), so uniqueness and routability are all the protocol needs.
* "fifo": exactly the numbering ONE reference scheduler would produce
  (`next_task_id++` in global FIFO order, task_dispatcher.cc:127): rank r must know how many
  requests EARLIER in the global queue were granted by other ranks, i.e. one all-reduce
  (sum) of the per-request grant flags per solve plus a local prefix sum.

Everything else (heartbeats, frees, keep-alives, ticks) is routed to the owning rank by
the caller-visible `owner_of_*` maps.

The class is backend-agnostic (any library speaking the ydsched C ABI) and
transport-agnostic (any torch.distributed backend), so the N>1 logic is tested on CPU
with gloo + the oracle and runs unchanged with NCCL on H100s.
"""
from __future__ import annotations

import zlib
from typing import Callable, Sequence

import numpy as np

from ._abi import (FILTER_OFFERED, GRANT8_DTYPE, GRANT_DTYPE, PACKED_IDS_DTYPE, REQ16_DTYPE, REQ_DTYPE, STAGE_CACHE,
                   STAGE_DEDUPE, STATUS_ENVIRONMENT_NOT_FOUND, STATUS_GRANTED)
from .dispatcher import Servant, TaskDispatcher


def default_digest_owner(digest: str, world: int) -> int:
    """Stable digest -> rank map.  Digests that co-occur on one servant must map to the
    same rank (they are one component); `keep_servant_alive` checks this."""
    return zlib.crc32(digest.encode()) % world


def component_digest_owner(servants: Sequence[Servant], world: int) -> Callable[[str, int], int]:
    """A digest -> rank map that keeps every component (digests joined through servants that hold several of them,
    the union-find of SyncTopology) on ONE rank: the owner is the default map applied to the component's smallest
    digest.  Digests no listed servant holds fall back to the default map.  Build it from the servant set the ranks
    agree on (all of them see every heartbeat) and pass it as `digest_owner`; with the plain default map a servant
    that advertises two compilers usually has digests on different ranks and `keep_servant_alive` refuses it."""
    parent: dict[str, str] = {}

    def find(x: str) -> str:
        parent.setdefault(x, x)
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for sv in servants:
        envs = list(sv.environments)
        for e in envs[1:]:
            a, b = find(envs[0]), find(e)
            if a != b:
                parent[max(a, b)] = min(a, b)
        if envs:
            find(envs[0])
    smallest: dict[str, str] = {}
    for d in list(parent):
        r = find(d)
        smallest[r] = min(smallest.get(r, d), d)

    def owner(digest: str, w: int) -> int:
        if digest in parent:
            return default_digest_owner(smallest[find(digest)], w)
        return default_digest_owner(digest, w)

    del world
    return owner


class ShardedDispatcher:
    def __init__(self, local: TaskDispatcher, rank: int, world: int, *, group=None, device=None,
                 digest_owner: Callable[[str, int], int] = default_digest_owner, id_mode: str = "strided"):
        """id_mode:
          "strided"  task id = local id * world + rank.  Needs `local` created with
                     id_stride=world, id_offset=rank (the library then hands out and accepts
                     such ids itself); no communication at all.  Ids are unique and routable
                     but not the single-scheduler numbering.
          "fifo"     exactly the ids one reference scheduler would hand out for the global
                     queue; costs one all-reduce of grant flags per solve."""
        assert id_mode in ("strided", "fifo")
        self.id_mode = id_mode
        self.local = local
        self.rank = rank
        self.world = world
        self.group = group
        self.device = device  # torch device for the collective (cuda:LOCAL_RANK with NCCL, cpu with gloo)
        self.digest_owner = digest_owner
        self.next_task_id = 0  # global id space
        # global task id -> local task id for the grants this rank owns: one chunk per solve
        # (global ids, local ids, alive flags), chunks ordered by first global id (ids only grow)
        self._chunks: list[list[np.ndarray]] = []
        self._owners_cache = None  # (owners array object, mine, mine on the collective's device)
        self.collective_bytes = 0

    # -- ownership -----------------------------------------------------------
    def owner_of_digest(self, digest: str) -> int:
        return self.digest_owner(digest, self.world)

    def owner_of_servant(self, servant: Servant) -> int:
        owners = {self.owner_of_digest(d) for d in servant.environments}
        if len(owners) > 1:
            raise ValueError(
                f"servant {servant.observed_location} holds digests owned by ranks {sorted(owners)}: "
                "the digest_owner map must keep a component on one rank"
            )
        return owners.pop() if owners else 0

    # -- servant maintenance ---------------------------------------------------
    def keep_servant_alive(self, servant: Servant, expires_in: float, *, now: float = 0.0) -> None:
        if self.owner_of_servant(servant) == self.rank:
            self.local.keep_servant_alive(servant, expires_in, now=now)

    def on_expiration_timer(self, *, now: float) -> None:
        self.local.on_expiration_timer(now=now)
        # "fifo" ids: leases that expired, were orphaned or swept never come back through free_tasks; once the library
        # holds no lease at all the whole id map is garbage
        if self._chunks and self.local.num_tasks() == 0:
            self._chunks = []

    # -- the hot path ------------------------------------------------------------
    def wait_for_starting_new_tasks(self, digests: Sequence[str], owners: np.ndarray, local_reqs: np.ndarray,
                                    now: float = 0.0) -> np.ndarray:
        """`owners[i]` = owning rank of global request i (or -1 if nobody holds its digest);
        `local_reqs` = REQ array of this rank's requests, in global order.  Returns a
        GRANT array for this rank's requests with GLOBAL task ids."""
        import torch
        import torch.distributed as dist

        del digests
        if self.id_mode == "strided":
            return self.local.wait_for_starting_new_tasks(local_reqs, now)
        if self._owners_cache is None or self._owners_cache[0] is not owners:
            mine = np.nonzero(owners == self.rank)[0]
            self._owners_cache = (owners, mine, torch.as_tensor(mine, device=self.device))
        _, mine, mine_t = self._owners_cache
        assert len(mine) == len(local_reqs)
        g = self.local.wait_for_starting_new_tasks(local_reqs, now).copy() if len(mine) else np.zeros(0, GRANT_DTYPE)
        ok = g["status"] == STATUS_GRANTED
        # the one exchange step: who was granted, over the whole global queue
        flags = torch.zeros(len(owners), dtype=torch.int32, device=self.device)
        if len(mine):
            flags[mine_t] = torch.as_tensor(ok.view(np.uint8)).to(self.device, non_blocking=True).to(torch.int32)
        if self.world > 1:
            dist.all_reduce(flags, op=dist.ReduceOp.SUM, group=self.group)
            self.collective_bytes += flags.numel() * 4
        csum = torch.cumsum(flags, 0)
        total = int(csum[-1].item()) if len(owners) else 0
        if len(mine):
            before = (csum - flags)[mine_t]  # grants strictly earlier in the global FIFO
            gids = np.uint64(self.next_task_id) + before.cpu().numpy().astype(np.uint64)
            if ok.any():
                self._chunks.append([gids[ok], g["task_id"][ok].copy(), np.ones(int(ok.sum()), dtype=bool)])
            g["task_id"][ok] = gids[ok]
        self.next_task_id += total
        return g

    def _lookup(self, global_ids):
        """Yields (chunk, positions in the chunk, positions in `global_ids`) for the ids this
        rank owns and still holds."""
        ids = np.asarray(global_ids, dtype=np.uint64)
        if not len(ids) or not self._chunks:
            return
        firsts = np.asarray([c[0][0] for c in self._chunks], dtype=np.uint64)
        which = np.searchsorted(firsts, ids, side="right").astype(np.int64) - 1
        for ci in np.unique(which[which >= 0]):
            gid, _, alive = self._chunks[ci]
            sel = np.nonzero(which == ci)[0]
            pos = np.searchsorted(gid, ids[sel])
            pos_c = np.minimum(pos, len(gid) - 1)
            hit = (pos < len(gid)) & (gid[pos_c] == ids[sel]) & alive[pos_c]
            if hit.any():
                yield self._chunks[ci], pos_c[hit], sel[hit]

    # -- lease maintenance, routed by global id -------------------------------------
    def free_tasks(self, global_ids) -> None:
        if self.id_mode == "strided":  # the library ignores ids that are not its own
            self.local.free_tasks(global_ids)
            return
        for chunk, pos, _ in self._lookup(global_ids):
            p = np.unique(pos)  # an id listed twice frees once (FreeTask of an unknown id is a no-op)
            self.local.free_tasks(chunk[1][p])
            chunk[2][p] = False
        self._chunks = [c for c in self._chunks if c[2].any()]

    def keep_tasks_alive(self, global_ids, new_expires_in: float, *, now: float = 0.0) -> np.ndarray:
        """Statuses for the ids this rank owns (False for ids owned elsewhere; the caller
        ORs the ranks' answers)."""
        if self.id_mode == "strided":
            return self.local.keep_tasks_alive(global_ids, new_expires_in, now=now)
        out = np.zeros(len(np.asarray(global_ids)), dtype=bool)
        for chunk, pos, where in self._lookup(global_ids):
            out[where] = self.local.keep_tasks_alive(chunk[1][pos], new_expires_in, now=now)
        return out


class RangeShardedDispatcher:
    """ONE scheduler whose pending queue is range-sharded over the GPUs of a node (include/ydshard.h;
    SURVEY.md 8(e) option 2, BASELINE.json north_star): rank g keeps the g-th contiguous FIFO range in
    its HBM, the servant table is replicated (every rank is fed the same heartbeats and ticks through
    the ordinary TaskDispatcher calls of `local`), and a solve makes exactly the decisions one
    TaskDispatcher would make on the concatenated queue.  The exchanges (class tables, per-class
    counts, reachable request records, per-servant claimed-slot counts) are NCCL collectives issued
    by the C++ library on its own stream; torch.distributed only carries the 128-byte ncclUniqueId
    here.  CUDA library only."""

    def __init__(self, local: TaskDispatcher, rank: int, world: int, *, device=None, group=None):
        import ctypes as C

        import torch
        import torch.distributed as dist

        from . import _abi

        self.local, self.rank, self.world = local, rank, world
        self.group = group
        lib = local._lib
        # Libraries without the NCCL path (the CPU oracles in the gloo tests): the same contract -- one queue cut into
        # per-rank ranges, replicated servant state, FIFO task ids, collective FreeTask -- with the exchange restated
        # over torch.distributed: the ranges are all-gathered and every rank decides the whole queue on its replica.
        self.native = hasattr(lib, "yd_shard_init")
        if not self.native:
            return
        buf = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)()
        if rank == 0 and lib.yd_shard_unique_id(buf) != 0:
            raise RuntimeError("yd_shard_unique_id failed (libnccl.so.2 not loadable?)")
        t = torch.tensor(list(buf), dtype=torch.uint8, device=device if dist.get_backend(group) == "nccl" else "cpu")
        dist.broadcast(t, src=0, group=group)
        uid = (C.c_uint8 * _abi.SHARD_UNIQUE_ID_BYTES)(*t.cpu().tolist())
        rc = lib.yd_shard_init(local._h, rank, world, uid)
        if rc != 0:
            raise RuntimeError(f"yd_shard_init failed: {rc}")

    def wait_for_starting_new_tasks(self, reqs_local, now: float, out=None):
        """Collective.  reqs_local: this rank's FIFO range (REQ_DTYPE), or an int n = the first n staged
        requests (TaskDispatcher.stage_requests).  Returns this rank's grants."""
        from .dispatcher import _ns

        lib, h = self.local._lib, self.local._h
        if not self.native:
            import torch.distributed as dist

            parts: list = [None] * self.world
            dist.all_gather_object(parts, np.ascontiguousarray(reqs_local), group=self.group)
            lo = sum(len(p) for p in parts[: self.rank])
            g = self.local.wait_for_starting_new_tasks(np.concatenate(parts), now)
            return g[lo:lo + len(reqs_local)].copy()
        if isinstance(reqs_local, (int, np.integer)):
            n, ptr = int(reqs_local), None
        else:
            assert reqs_local.dtype == REQ_DTYPE and reqs_local.flags.c_contiguous
            n, ptr = reqs_local.shape[0], reqs_local.ctypes.data
        if out is None:
            out = np.zeros(max(n, 1), dtype=GRANT_DTYPE)
        rc = lib.yd_shard_wait_for_starting_new_tasks(h, _ns(now), ptr, n, out.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"yd_shard_wait_for_starting_new_tasks failed: {rc}")
        return out[:n]

    def wait_for_starting_new_tasks_packed(self, reqs16_local, now: float, out=None):
        """Collective, over the packed interface (yd_shard_wait_for_starting_new_tasks_packed): reqs16_local is this
        rank's FIFO range (REQ16_DTYPE, `pack_requests`), or an int n = the first n staged requests (24-byte records,
        TaskDispatcher.stage_requests).  Returns (GRANT8 array, PACKED_IDS record) as
        TaskDispatcher.wait_for_starting_new_tasks_packed(unpack=False) does; the ordinals count the grants of the
        whole group's batch, so `unpack_grants` gives what wait_for_starting_new_tasks returns."""
        from .dispatcher import _ns

        lib, h = self.local._lib, self.local._h
        if not self.native:
            import torch.distributed as dist

            parts: list = [None] * self.world
            dist.all_gather_object(parts, np.ascontiguousarray(reqs16_local), group=self.group)
            lo = sum(len(p) for p in parts[: self.rank])
            g8, ids = self.local.wait_for_starting_new_tasks_packed(np.concatenate(parts), now, unpack=False)
            return g8[lo:lo + len(reqs16_local)].copy(), ids
        if isinstance(reqs16_local, (int, np.integer)):
            n, ptr = int(reqs16_local), None
        else:
            assert reqs16_local.dtype == REQ16_DTYPE and reqs16_local.flags.c_contiguous
            n, ptr = reqs16_local.shape[0], reqs16_local.ctypes.data
        if out is None:
            out = np.zeros(max(n, 1), dtype=GRANT8_DTYPE)
        assert out.dtype == GRANT8_DTYPE and out.shape[0] >= n and out.flags.c_contiguous
        ids = np.zeros(1, dtype=PACKED_IDS_DTYPE)
        rc = lib.yd_shard_wait_for_starting_new_tasks_packed(h, _ns(now), ptr, n, out.ctypes.data, ids.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"yd_shard_wait_for_starting_new_tasks_packed failed: {rc}")
        return out[:n], ids[0]

    def free_tasks(self, ids) -> None:
        """Collective FreeTask: every rank passes the ids it wants released (its own grants, typically)."""
        ids = np.ascontiguousarray(np.asarray(ids, dtype=np.uint64))
        if not self.native:
            import torch.distributed as dist

            parts: list = [None] * self.world
            dist.all_gather_object(parts, ids, group=self.group)
            self.local.free_tasks(np.concatenate(parts))  # every replica holds every lease
            return
        rc = self.local._lib.yd_shard_free_tasks(self.local._h, ids.ctypes.data if len(ids) else None, len(ids))
        if rc != 0:
            raise RuntimeError(f"yd_shard_free_tasks failed: {rc}")

    # -- replicated calls (ydshard.h): every rank makes the call with the same arguments and gets the single scheduler's
    # answer.  Over gloo with the CPU libraries every replica holds every lease, so these are the local calls there.
    def keep_tasks_alive(self, ids, new_expires_in, *, now: float = 0.0) -> np.ndarray:
        """Replicated KeepTaskAlive: the holder of each lease renews it; every rank returns the same flags.
        `new_expires_in` is one lease length, or one per id (yd_shard_keep_tasks_alive)."""
        if not self.native:
            return self.local.keep_tasks_alive(ids, new_expires_in, now=now)
        return self.local._keep_alive_with(self.local._lib.yd_shard_keep_task_alive, ids, new_expires_in, now,
                                           fn_each=self.local._lib.yd_shard_keep_tasks_alive)

    def notify_servants_running_tasks(self, batch) -> list[list[int]]:
        """Replicated NotifyServantRunningTasks for [(location, tasks)]: an id is unknown iff no rank holds its lease."""
        if not self.native:
            return self.local.notify_servants_running_tasks(batch)
        return self.local._notify_with(self.local._lib.yd_shard_notify_servants_running_tasks, batch)

    def get_running_tasks(self):
        """Replicated GetRunningTasks: the whole group's list, in the single scheduler's order."""
        if not self.native:
            return self.local.get_running_tasks()
        return self.local._running_with(self.local._lib.yd_shard_get_running_tasks)

    def running_index_refresh(self) -> int:
        """Replicated RunningTaskKeeper::Refresh: afterwards `local.find_running_tasks` answers for the whole group."""
        if not self.native:
            return self.local.running_index_refresh()
        return int(self.local._lib.yd_shard_running_index_refresh(self.local._h))

    def wait_for_starting_task_rpcs(self, rpcs: np.ndarray, now: float = 0.0):
        """Replicated window of WaitForStartingTask RPCs: every rank passes the whole window and gets (results, grants)
        for all of it; each rank decides an even share of the expanded queue."""
        if not self.native:
            return self.local.wait_for_starting_task_rpcs(rpcs, now)
        return self.local._rpcs_with(self.local._lib.yd_shard_wait_for_starting_task_rpcs, rpcs, now)

    def wait_for_starting_task_rpcs_packed(self, rpcs: np.ndarray, now: float = 0.0):
        """Replicated wait_for_starting_task_rpcs with 8-byte grants (yd_shard_wait_for_starting_task_rpcs_packed):
        every rank gets the same (results, GRANT8 array, PACKED_IDS record) for the whole window."""
        if not self.native:
            return self.local.wait_for_starting_task_rpcs_packed(rpcs, now)
        return self.local._rpcs_packed_with(self.local._lib.yd_shard_wait_for_starting_task_rpcs_packed, rpcs, now)

    # -- the pre-filtered solve (BASELINE configs[3]): each rank filters its own range, then the group decides the
    # concatenation of the offered ranges.  Both return this rank's (verdicts, hits, grants of its offered requests).
    def filter_and_wait_for_starting_new_tasks(self, reqs_local: np.ndarray, cache_keys=None, task_digests=None,
                                               now: float = 0.0):
        """Collective TaskDispatcher.filter_and_wait_for_starting_new_tasks over the queue the ranks' ranges make:
        cache_keys / task_digests are this rank's requests' keys (the same kinds on every rank)."""
        if not self.native:
            km = None if cache_keys is None else TaskDispatcher._key_matrix(cache_keys)
            dm = None if task_digests is None else TaskDispatcher._key_matrix(task_digests)
            parts = self._gather((np.ascontiguousarray(reqs_local), km, dm))

            def keys(j):  # (None: no rank passed keys of this kind, or the whole queue is empty)
                ms = [p[j][:len(p[0])] for p in parts if p[j] is not None and len(p[0])]
                return np.concatenate(ms) if ms else None
            whole = self.local.filter_and_wait_for_starting_new_tasks(np.concatenate([p[0] for p in parts]), keys(1), keys(2),
                                                                      now)
            return self._my_slice([len(p[0]) for p in parts], *whole)
        return self.local._filter_with(self.local._lib.yd_shard_filter_and_wait_for_starting_new_tasks, reqs_local,
                                       cache_keys, task_digests, now, None, None, True)

    def filter_and_wait_for_starting_new_tasks_packed(self, reqs16_local: np.ndarray, cache_digests=None, task_digests=None,
                                                      now: float = 0.0, hits: bool = False):
        """Collective TaskDispatcher.filter_and_wait_for_starting_new_tasks_packed over the queue the ranks' ranges make
        (yd_shard_filter_and_wait_for_starting_new_tasks_packed): this rank's (verdicts, hits or None, GRANT8 of its
        offered requests, PACKED_IDS record); the ordinals count the grants of the group's whole offered queue, and the
        ids are the same on every rank."""
        if not self.native:
            digests = lambda d: None if d is None else np.ascontiguousarray(d, dtype=np.uint8).reshape(-1, 32)  # noqa: E731
            parts = self._gather((np.ascontiguousarray(reqs16_local), digests(cache_digests), digests(task_digests)))

            def keys(j):  # (None: no rank passed digests of this kind, or the whole queue is empty)
                ms = [p[j][:len(p[0])] for p in parts if p[j] is not None and len(p[0])]
                return np.concatenate(ms) if ms else None
            v, h, g8, ids = self.local.filter_and_wait_for_starting_new_tasks_packed(
                np.concatenate([p[0] for p in parts]), keys(1), keys(2), now, hits)
            return (*self._my_slice([len(p[0]) for p in parts], v, h, g8), ids)
        return self.local._filter_packed_with(self.local._lib.yd_shard_filter_and_wait_for_starting_new_tasks_packed,
                                              reqs16_local, cache_digests, task_digests, now, hits, None, None)

    def derive_filter_and_wait_for_starting_new_tasks(self, reqs_local: np.ndarray, src_local,
                                                      stages: int = STAGE_CACHE | STAGE_DEDUPE, now: float = 0.0):
        """Collective TaskDispatcher.derive_filter_and_wait_for_starting_new_tasks: src_local (a TaskSources with its
        own argument table) describes this rank's range.  If any rank's descriptors are refused, every rank raises
        (TaskKeysError on the ranks whose own descriptors were refused) and nothing is decided."""
        from .dispatcher import TaskKeysError, TaskSources

        if not self.native:
            parts = self._gather((np.ascontiguousarray(reqs_local), src_local))
            counts = [len(p[0]) for p in parts]
            try:
                whole = self.local.derive_filter_and_wait_for_starting_new_tasks(
                    np.concatenate([p[0] for p in parts]), TaskSources.concat([p[1] for p in parts], counts), stages, now)
            except TaskKeysError:
                # this rank's own descriptors refused: raises TaskKeysError with its code
                self.local.derive_task_keys(reqs_local, src_local, cache_keys=False, task_digests=False)
                raise RuntimeError("the pre-filtered solve was refused: another rank's descriptors") from None
            return self._my_slice(counts, *whole)
        return self.local._derive_filter_with(self.local._lib.yd_shard_derive_filter_and_wait_for_starting_new_tasks,
                                              reqs_local, src_local, stages, now, None, None, True)

    def _gather(self, obj) -> list:
        import torch.distributed as dist

        parts: list = [None] * self.world
        dist.all_gather_object(parts, obj, group=self.group)
        return parts

    def _my_slice(self, counts, verdicts, hits, grants):
        """This rank's part of a single handle's pre-filtered solve over the concatenated queue."""
        lo = sum(counts[: self.rank])
        hi = lo + counts[self.rank]
        first = int((verdicts[:lo] == FILTER_OFFERED).sum())
        mine = int((verdicts[lo:hi] == FILTER_OFFERED).sum())
        return verdicts[lo:hi].copy(), None if hits is None else hits[lo:hi].copy(), grants[first:first + mine].copy()

    def export_state(self, now: float = 0.0) -> bytes:
        """Collective.  The group's state as ONE scheduler's export (ydstate.h), the same bytes on every rank: a
        single TaskDispatcher, or a group of any size, can import it (import_state)."""
        import ctypes as C

        from .dispatcher import _ns

        if not self.native:
            return self.local.export_state(now)  # every replica holds every lease
        lib, h, t = self.local._lib, self.local._h, _ns(now)
        n = lib.yd_shard_export_state(h, t, None, 0)
        if n == 0:
            raise RuntimeError("yd_shard_export_state: the ranks' replicated state disagrees")
        buf = C.create_string_buffer(n)
        m = lib.yd_shard_export_state(h, t, buf, n)
        assert m == n, (m, n)
        return buf.raw

    def import_state(self, blob: bytes, now: float = 0.0) -> None:
        """Collective.  Load an export (of a single handle or of a group of any size) into this group of fresh
        handles.  All or nothing: if any rank refuses, every rank raises StateError with the same code and stays
        fresh."""
        from . import _abi
        from .dispatcher import StateError, TaskDispatcher, _ns

        data = bytes(blob)
        if self.native:
            rc = self.local._lib.yd_shard_import_state(self.local._h, _ns(now), data, len(data))
            if rc != _abi.STATE_OK:
                raise StateError(rc)
            return
        import hashlib

        import torch.distributed as dist

        # Every refusal leaves a handle fresh, but a success does not: check on a scratch handle of the same library
        # and config first, so that the local import runs only where every rank will succeed.  An empty blob is
        # refused as not fresh, or as malformed by a fresh handle.
        rc = _abi.STATE_OK
        try:
            self.local.import_state(b"", now)
        except StateError as e:
            rc = e.code if e.code == _abi.STATE_NOT_FRESH else _abi.STATE_OK
        if rc == _abi.STATE_OK:
            scratch = TaskDispatcher(self.local._lib, **self.local._config)
            try:
                scratch.import_state(data, now)
            except StateError as e:
                rc = e.code
            finally:
                scratch.close()
        verdicts: list = [None] * self.world
        dist.all_gather_object(verdicts, (rc, hashlib.sha256(data).digest()), group=self.group)
        for code, digest in verdicts:
            if code == _abi.STATE_OK and digest != verdicts[0][1]:
                code = _abi.STATE_BAD_BLOB
            if code != _abi.STATE_OK:
                raise StateError(code)
        self.local.import_state(data, now)

    def last_stats(self) -> dict | None:
        import ctypes as C

        from . import _abi

        if not self.native:
            return None
        st = _abi.yd_shard_stats()
        if not self.local._lib.yd_shard_last_stats(self.local._h, C.byref(st)):
            return None
        return {"total_ms": st.total_ms, "exchange_ms": list(st.exchange_ms), "exchange_bytes": list(st.exchange_bytes),
                "decisions_local": st.decisions_local, "granted_local": st.granted_local, "granted_total": st.granted_total,
                "merge_rounds": st.merge_rounds, "kernel_launches": st.kernel_launches}

    def close(self) -> None:
        if self.native:
            self.local._lib.yd_shard_finalize(self.local._h)
