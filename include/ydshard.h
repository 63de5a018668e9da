/* ydshard.h -- ONE scheduler whose pending queue is range-sharded over the GPUs of a node.
 *
 * BASELINE.json north_star / SURVEY.md 8(e) option 2: the FIFO queue is cut into `world` contiguous
 * ranges, rank g keeps range g in its HBM; the servant table (<= 288 KB) and all scheduler state
 * that decisions depend on (running_tasks per servant) are REPLICATED: every rank receives the same
 * heartbeats / expiration ticks through the ordinary calls of ydsched.h.  A solve produces exactly the
 * decisions of one TaskDispatcher fed the concatenated queue (task_dispatcher.cc:93-140; the coupling
 * that must survive the sharding is `++running_tasks` at :123-124).  Per solve the ranks exchange, over
 * NCCL (NVLink / NVSwitch):
 *
 *   1. all-gather   the class tables (which (digest, min_version) classes occur, 16 KB per rank)
 *   2. all-gather   per-class request counts  -> every request's FIFO rank inside its class
 *   3. all-reduce   the per-class request records the slot lists can reach (a disjointly written
 *                   buffer: an all-gather-v; <= one 8-byte record per (class, eligible slot))
 *   4. all-reduce   the per-servant claimed-slot counts (u32[S]) + per-rank grant counts + flags
 *
 * Between 3 and 4 every rank runs the same slot-side merge (solve_merge.cuh) on the same data and
 * keeps the verdicts of its own requests.  Task ids are the batch's FIFO ordinals (rank g's grants
 * follow those of the lower ranks).  Leases (TaskDesc, task_dispatcher.h:199-215) live on the rank
 * that holds the request, so a zombie swept by a heartbeat or a freed lease lowers running_tasks on
 * that rank first; each rank counts those decrements and the next collective call (exchange 1 of a
 * solve, or yd_shard_free_tasks) hands them to the others.  After every collective call every rank's
 * running_tasks is the single scheduler's; in between, a non-holder rank's may be higher.
 *
 * The library dlopen()s libnccl.so.2 on yd_shard_init: a single-GPU process never needs it.
 */
#ifndef YDSHARD_H_
#define YDSHARD_H_

#include "ydfilter_packed.h"
#include "ydkeys.h"
#include "ydrpcs_packed.h"
#include "ydsched.h"
#include "ydservice.h"

#ifdef __cplusplus
extern "C" {
#endif

#define YD_SHARD_UNIQUE_ID_BYTES 128

/* Rank 0: a fresh ncclUniqueId to hand to every rank (any transport: a file, MPI, torch.distributed).
 * Returns 0, or non-zero if NCCL cannot be loaded. */
int yd_shard_unique_id(uint8_t out[YD_SHARD_UNIQUE_ID_BYTES]);

/* Collective: joins `s` (one handle per process, on its own GPU) to a communicator of `world` ranks. */
int yd_shard_init(yd_sched* s, int rank, int world, const uint8_t unique_id[YD_SHARD_UNIQUE_ID_BYTES]);
void yd_shard_finalize(yd_sched* s);

/* Collective, THE HOT PATH: the whole queue = ranks' `reqs_local` concatenated in rank order.  out_local[i]
 * is what the i-th request of this rank's range gets (same fields as yd_wait_for_starting_new_tasks;
 * task ids number the grants of the whole batch in FIFO order).  reqs_local == NULL: the range staged with
 * yd_stage_requests.  A batch with a component that needs the sequential solver (several servants behind one
 * requestor IP, more than 32 classes on one component, the last-resort rule, a request beyond the exchange-3
 * margin) is decided by every rank: the ranges are gathered and every rank runs the ordinary solve on the
 * whole queue, keeping its own range's grants and leases.  Returns 0; 1 (on every rank, nothing exchanged or
 * changed) if the cluster has capacities above 8192 per servant, or if reqs_local == NULL and n_local is
 * larger than the staged queue. */
int yd_shard_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs_local, size_t n_local,
                                         yd_grant* out_local);

/* Collective: the same call over the packed interface (yd_wait_for_starting_new_tasks_packed, ydsched.h): 16-byte
 * requests up and 8-byte grants down on every rank.  It is yd_shard_wait_for_starting_new_tasks on the unpacked
 * requests (yd_unpack_req) -- the same queue, the same four exchanges, the same decisions -- with the grants packed:
 * out_local[i] belongs to the i-th request of this rank's range, and its ordinal counts the grants of the WHOLE group's
 * batch in FIFO order, so yd_unpack_grant(out_local[i], *ids) is, field for field, what the unpacked call returns for
 * that request.  *ids (may be NULL) is the same on every rank, the group batch's first task id and the stride, and is
 * valid even if nothing was granted.  reqs_local == NULL: the range staged with yd_stage_requests (24-byte records),
 * decided with packed grants; afterwards the staging area follows the unpacked call's rules.  Returns 0; 1 (on every
 * rank, nothing decided, no state changed) where the unpacked call refuses, and if the group's queue -- the ranges'
 * lengths summed, known after the first exchange -- is longer than 2^30 requests (the ordinal has 30 bits). */
int yd_shard_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs_local,
                                                size_t n_local, yd_grant8* out_local, yd_packed_ids* ids);

/* Collective FreeTask x n (task_dispatcher.cc:167-188): every rank passes the ids IT wants freed (any
 * subset, also none, also ids another rank holds); the ids are gathered, a lease is released by the rank
 * that holds it and the running_tasks decrements reach every replica through one all-reduce. */
int yd_shard_free_tasks(yd_sched* s, const uint64_t* ids, size_t n);

/* STATE HANDOVER (include/ydstate.h, format version 1).  A group exports and imports as ONE scheduler: the export of
 * a group is byte for byte what a single handle fed the concatenated queue (the same calls, the same interning)
 * exports, and any version-1 export -- of a single handle, or of a group of any size -- imports into a group of any
 * size, so a restart may also change the number of GPUs.  yd_export_state / yd_import_state refuse sharded handles
 * (0 / YD_STATE_UNSUPPORTED): a lease lives on one rank, so no rank alone holds the state.
 *
 * Collective.  The export of the whole group.  Every rank returns the same size and, where out / cap allow, writes
 * the same bytes (out may be NULL with cap 0 to ask for the size; that query is a collective call too).  Changes
 * nothing: the group's later decisions are those it would have made without it.  Returns 0 on every rank if the
 * ranks' replicated state (servants, intern tables, next task id, the bookkeeper's groups) disagrees, which is a bug
 * and is reported on stderr. */
size_t yd_shard_export_state(yd_sched* s, int64_t now_ns, uint8_t* out, size_t cap);

/* Collective.  Loads a version-1 export into a group of fresh handles (yd_create, yd_shard_init, nothing else).
 * Returns YD_STATE_* (ydstate.h), the SAME code on every rank.  All or nothing: if any rank refuses (not fresh, a
 * config mismatch, no memory, a malformed blob, or a blob that differs from rank 0's: YD_STATE_BAD_BLOB), every rank
 * returns the refusal of the lowest such rank and stays fresh.  Lease k of the export's n (ascending id order) goes
 * to rank k * world / n; every rank's running_tasks counts every lease; a bookkeeper entry goes to the rank holding
 * its task_grant_id's lease (rank 0 if there is none). */
int yd_shard_import_state(yd_sched* s, int64_t now_ns, const uint8_t* blob, size_t len);

/* REPLICATED CALLS: the rest of TaskDispatcher, and SchedulerServiceImpl, answered by the group as ONE scheduler.
 * Every rank makes the call with the same arguments, in the same order relative to the other calls on its handle (the
 * conditions under which a front end feeds every rank the same heartbeats); every rank then returns the same answer,
 * and it is what one handle fed the concatenated queue returns for the same call.  Arguments are not checked across
 * ranks: ranks that pass different ones get answers that match no single scheduler.  Each call makes one exchange
 * (GetRunningTasks two, WaitForStartingTask one more than its solve) and the running_tasks decrements a rank has not
 * shared yet ride along it, so the invariant above holds after each.  On a handle that has not joined a group, the
 * calls that return a count are the single-handle call.  The per-rank calls of ydsched.h (yd_keep_task_alive,
 * yd_notify_*, yd_get_running_tasks, yd_running_index_refresh, yd_wait_for_starting_task_rpcs) keep answering for the
 * rank's own leases only.
 *
 * KeepTaskAlive x n.  The holder of a lease renews it, the other ranks answer 0; one sum all-reduce of a u32 flag per
 * id and the decrements.  Returns 0; 1 (nothing exchanged) if the handle has not joined a group or n >= 2^30. */
int yd_shard_keep_task_alive(yd_sched* s, int64_t now_ns, const uint64_t* task_ids, size_t n, int64_t new_expires_in_ns,
                             uint8_t* ok_out);
/* KeepTaskAlive x n with a lease length per id, as yd_keep_tasks_alive (the last occurrence of an id sets its expiry);
 * the same one all-reduce and return values as yd_shard_keep_task_alive, which is its case of one length. */
int yd_shard_keep_tasks_alive(yd_sched* s, int64_t now_ns, const uint64_t* task_ids, const int64_t* new_expires_in_ns,
                              size_t n, uint8_t* ok_out);
/* NotifyServantRunningTasks x n, as yd_notify_servants_running_tasks.  Each rank sweeps and checks its own leases; one
 * sum all-reduce of a u32 word per reported id (rank + 1 where permitted) and the decrements.  An id is unknown iff no
 * rank permits it.  Each rank's bookkeeper keeps the tasks whose lease it holds. */
size_t yd_shard_notify_servants_running_tasks(yd_sched* s, const yd_heartbeat_item* items, size_t n, uint64_t* unknown_out,
                                              size_t* unknown_counts);
/* GetRunningTasks, in the single scheduler's order.  Two all-gathers: the packed bookkeepers' lengths with the
 * decrements, then the bookkeepers, merged by each task's position in the heartbeat that reported it.  The strings stay
 * valid until the next call that mutates the handle. */
size_t yd_shard_get_running_tasks(yd_sched* s, yd_running_task* out, size_t cap);
/* RunningTaskKeeper::Refresh over the group: the snapshot is yd_shard_get_running_tasks' list, so yd_running_index_find
 * and yd_running_index_entry on any rank then answer for the whole group. */
size_t yd_shard_running_index_refresh(yd_sched* s);
/* WaitForStartingTask x n_rpcs, as yd_wait_for_starting_task_rpcs (the same expansion, limits and return values).  The
 * expanded queue is cut into `world` even contiguous ranges; each rank expands its own and decides it with
 * yd_shard_wait_for_starting_new_tasks, and one all-gather (a grant is 4 u32 words, padded to the longest range) gives
 * every rank the whole window's decisions, to which it applies the stop rules.  A refusal ((size_t)-1: cap too small, a
 * batch above 2^30 decisions, or capacities above 8192 per servant) happens on every rank and decides nothing. */
size_t yd_shard_wait_for_starting_task_rpcs(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs,
                                            yd_rpc_wait_result* results, yd_grant* grants_out, size_t cap);
/* yd_shard_wait_for_starting_task_rpcs with 8-byte grants (ydrpcs_packed.h): defined as that call, then yd_pack_grant of
 * every grant with the group batch's *ids (the same on every rank).  Every rank returns the same results, grants and
 * *ids, and its refusals (those of the unpacked group call, and of yd_wait_for_starting_task_rpcs_packed) happen on every
 * rank.  Every rank expands its own even range of the window on the device, decides it with the packed sharded solve,
 * and one all-gather of the 8-byte grants (device to device) gives every rank the whole window to report.  On a handle
 * that has not joined a group, this is the single-handle call. */
size_t yd_shard_wait_for_starting_task_rpcs_packed(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs,
                                                   yd_rpc_wait_result* results, yd_grant8* grants_out, size_t cap,
                                                   yd_packed_ids* ids);
/* A SchedulerServiceImpl over the group (ydservice.h; ydwire.h works on it unchanged).  Collective; every rank passes the
 * same config.  Its handlers make the replicated calls above: Heartbeat's notification, WaitForStartingTask,
 * KeepTaskAlive, GetRunningTasks, and FreeTask through yd_shard_free_tasks (rank 0 passes the ids).  KeepServantAlive is
 * the per-rank call, fed to every rank alike.  The serving-daemon tokens are rank 0's, through one all-gather at
 * creation and one per roll-out.  Fed the same calls, every rank's service returns the same answers (and the wire
 * layer writes the same bytes).  Returns NULL on every rank if the handle has not joined a group or the config is
 * refused (as yd_service_create). */
yd_service* yd_shard_service_create(yd_sched* s, int64_t now_ns, const yd_service_config* cfg);

/* THE PRE-FILTERED SOLVE OVER A GROUP (BASELINE configs[3]; yd_filter_and_wait_for_starting_new_tasks, ydsched.h, and
 * yd_derive_filter_and_wait_for_starting_new_tasks, ydkeys.h).  Collective: the whole queue is the ranks' `reqs_local`
 * concatenated in rank order, as in yd_shard_wait_for_starting_new_tasks.  Each rank runs the filter stages (the key
 * derivation, the bloom probe, the in-flight index probe and the order-keeping compaction) on its own range on its own
 * GPU, then every rank enters the sharded solve with its offered requests, also a rank whose range is empty or filtered
 * out entirely.  The answers equal those of one handle given the concatenated queue through the single-handle call:
 * verdict_out[i] and hits_out[i] (may be NULL) belong to the i-th request of this rank's range; grants_out[0 .. returned)
 * are the grants of this rank's OFFERED requests, in order; task ids number the grants of the group's whole offered queue
 * in FIFO order; afterwards every replica's running_tasks and next task id are the single handle's.  Returns how many of
 * this rank's requests were offered.
 *
 * Not checked across ranks, as in the other replicated calls: the bloom filters (each rank probes its own, so the ranks
 * hold the same one: yd_bloom_reset / yd_bloom_load / yd_bloom_add fed alike) and the in-flight index (hits_out[i].
 * snapshot_index refers to the group snapshot when it was last refreshed with yd_shard_running_index_refresh on every
 * rank).  Programmer errors abort as in the single-handle calls (a bloom filter used before yd_bloom_reset / _load, keys
 * longer than the bloom filter takes, more than 2^30 requests).
 *
 * Afterwards each rank's staging area holds exactly its offered requests, in order (none if it offered none), so
 * yd_shard_wait_for_starting_new_tasks(s, now, NULL, offered, out) decides them again.  A refusal returns (size_t)-1 on
 * every rank and decides nothing: capacities above 8192 per servant (replicated state: every rank sees it before any
 * stage, and the staged queues are kept), or the sharded solve's own refusals (then after the stages: the staging areas
 * hold the offered requests).  On a handle that has not joined a group, these are the single-handle calls.
 *
 * yd_last_solve_stats then reports the rank's stages: prep_ms (= total_ms) is their device time (derivation, filter
 * stages, compaction), decisions = n_local, granted = this rank's grants; yd_shard_last_stats describes the solve. */
size_t yd_shard_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs_local,
                                                       size_t n_local, const yd_prefilter* filter, uint8_t* verdict_out,
                                                       yd_running_hit* hits_out, yd_grant* grants_out);
/* The same from task descriptors: each rank's `src_local` describes its own range with its own argument table, and the
 * equivalent single-handle queue appends the ranks' argument tables in rank order, each rank's args_index shifted by the
 * earlier ranks' n_args (the ranks pass the same source_digest_len, which is not checked).  `stages` is YD_STAGE_* and
 * must be the same on every rank.  If any rank's descriptors are refused (a YD_KEYS_* code of yd_derive_task_keys), every
 * rank returns (size_t)-1, decides nothing and keeps its staged queue: the ranks agree on this through one small
 * all-gather before anything is uploaded.  The keys each request needs depend on that request alone, so the derivation,
 * the call's most expensive stage, is split over the GPUs with the ranges. */
size_t yd_shard_derive_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs_local,
                                                              size_t n_local, const yd_task_sources* src_local,
                                                              uint32_t stages, uint8_t* verdict_out,
                                                              yd_running_hit* hits_out, yd_grant* grants_out);
/* The same over the packed interface (yd_filter_and_wait_for_starting_new_tasks_packed, ydsched.h): defined as
 * yd_shard_filter_and_wait_for_starting_new_tasks on the unpacked requests and the hex-expanded keys, with the grants
 * packed as yd_shard_wait_for_starting_new_tasks_packed packs them: their ordinals count the grants of the group's whole
 * offered queue, and *ids (may be NULL) is the same on every rank and valid even if nothing was offered.  Its refusals
 * are the unpacked call's, and a group queue of offered requests above 2^30 (the packed solve's); each returns
 * (size_t)-1 on every rank.  On a handle that has not joined a group, this is the single-handle call. */
size_t yd_shard_filter_and_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs_local,
                                                              size_t n_local, const yd_prefilter_packed* filter,
                                                              uint8_t* verdict_out, yd_running_hit* hits_out,
                                                              yd_grant8* grants_out, yd_packed_ids* ids);

/* Device time (ms, CUDA events on the solve stream) of the last sharded solve's phases: local kernels and
 * the four exchanges.  Returns 0 if there was none. */
typedef struct yd_shard_stats {
  float total_ms;       /* first kernel .. grants ready on the device */
  float exchange_ms[4]; /* the four NCCL exchanges, including waiting for the slowest rank */
  uint64_t exchange_bytes[4];
  uint64_t decisions_local, granted_local, granted_total;
  uint32_t merge_rounds, kernel_launches;
} yd_shard_stats;
int yd_shard_last_stats(yd_sched* s, yd_shard_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* YDSHARD_H_ */
