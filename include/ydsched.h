/*
 * ydsched.h -- C ABI of the H100-native yadcc scheduler hot path.
 *
 * This is the drop-in boundary (SURVEY.md 8(b)): every entry point below
 * replaces one public method of the reference's `TaskDispatcher`
 * (yadcc/scheduler/task_dispatcher.h:120-181), which in production is called
 * only from `SchedulerServiceImpl` (yadcc/scheduler/scheduler_service_impl.cc:
 * 171,180,235,255,292,308,315).  No C++ or torch types cross this boundary:
 * plain pointers, sizes and fixed-width integers only.
 *
 * Three shared libraries export exactly this ABI:
 *   - yadcc_b200/libydsched.so        host C++ + sm_90a CUDA kernels (the product)
 *   - oracle/libydoracle.so           CPU restatement of the algorithm (test infra)
 *   - oracle/_ref/libydref.so         the reference's own .cc files compiled
 *                                     verbatim against oracle/shim (test infra)
 *
 * Conventions (mirroring the reference, task_dispatcher.h / .cc):
 *   - Time never comes from a wall clock inside the library.  Every call that
 *     reads `flare::ReadCoarseSteadyClock()` in the reference takes `now_ns`
 *     (steady-clock nanoseconds) here, so event streams replay bit-exactly.
 *   - The 1 Hz `OnExpirationTimer` (task_dispatcher.cc:81-82,498-536) is driven
 *     by the caller through `yd_on_expiration_timer`.
 *   - Calls on one handle must be externally serialised, which is what the
 *     reference's single `allocation_lock_` (task_dispatcher.h:289) does.
 *   - Errors are values (status codes / counts / flags).  Programmer errors
 *     (NULL handle, invariant violations the reference FLARE_CHECKs) abort.
 *   - All strings are borrowed for the duration of the call only.
 *   - Integer field widths are the wire widths of yadcc/api/scheduler.proto
 *     (HeartbeatRequest :64-120, all uint32 except memory which is uint64).
 */
#ifndef YDSCHED_H_
#define YDSCHED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YD_ABI_VERSION 1u

/* WaitStatus numeric values are the reference's (task_dispatcher.h:41-44);
 * 2 is the success arm of flare::Expected<TaskAllocation, WaitStatus>. */
#define YD_STATUS_ENVIRONMENT_NOT_FOUND 0u
#define YD_STATUS_TIMEOUT 1u
#define YD_STATUS_GRANTED 2u

/* ServantPriority, yadcc/api/scheduler.proto:38-48. */
#define YD_PRIORITY_UNKNOWN 0
#define YD_PRIORITY_DEDICATED 1
#define YD_PRIORITY_USER 2

#define YD_REQ_FLAG_PREFETCH 1u /* `prefetching` arg, task_dispatcher.cc:96 */

#define YD_NO_SERVANT 0xffffffffu
#define YD_IP_NONE 0u /* requestor IP that was never seen as a servant IP */

typedef struct yd_sched yd_sched; /* opaque; one per scheduler process */

typedef struct yd_config {
  uint32_t abi_version; /* must be YD_ABI_VERSION */
  int32_t device;       /* CUDA device ordinal; ignored by the CPU oracles */
  /* gflag --servant_min_memory_for_accepting_new_task (task_dispatcher.cc:35-38),
   * parsed with yd_parse_size; NULL means the reference default "10G". */
  const char* servant_min_memory_for_accepting_new_task;
  /* Solver selection for the CUDA backend: 0 = auto, 1 = row-scan solver,
   * 2 = slot-stream solver.  Ignored by the oracles. */
  uint32_t solver;
  /* bit 0: CUDA backend launches the solve kernel by kernel instead of replaying a
   * captured CUDA graph, so yd_solve_stats can split prep / solve / final. */
  uint32_t reserved;
  /* Sharded deployments (one handle per GPU, yadcc_b200/sharded.py): task ids handed out
   * and accepted by this handle are local_id * id_stride + id_offset, so N shards share one
   * id space without talking to each other.  0 means stride 1, offset 0 (the reference's
   * numbering).  Ignored by the oracles. */
  uint32_t id_stride;
  uint32_t id_offset;
} yd_config;

/* ServantPersonality, task_dispatcher.h:80-116, as filled in by
 * SchedulerServiceImpl::Heartbeat (scheduler_service_impl.cc:124-170). */
typedef struct yd_servant {
  int32_t version;                   /* int in the reference (h:84) */
  int32_t priority;                  /* YD_PRIORITY_* (h:112) */
  int32_t not_accepting_task_reason; /* NotAcceptingTaskReason (h:115) */
  uint32_t num_envs;
  const char* observed_location; /* "ip:port" as seen by the scheduler (h:87) */
  const char* reported_location; /* "ip:port" as reported (h:91) */
  const char* const* env_digests; /* num_envs compiler digests (h:94) */
  uint32_t num_processors;        /* h:97 */
  uint32_t current_load;          /* h:100 */
  uint32_t max_tasks;             /* h:109 ("capacity" on the wire) */
  uint32_t reserved;
  uint64_t total_memory_in_bytes;     /* h:103 */
  uint64_t memory_available_in_bytes; /* h:106 */
} yd_servant;

/* One WaitForStartingNewTask call (task_dispatcher.cc:93-96): the
 * TaskPersonality (h:48-66) with its two strings replaced by interned ids,
 * plus `expires_in` and `prefetching`.  24 bytes. */
typedef struct yd_task_req {
  uint32_t env_id;       /* yd_intern_env(env_desc.compiler_digest) */
  uint32_t min_version;  /* TaskPersonality::min_version */
  uint32_t requestor_ip; /* yd_intern_ip(TaskPersonality::requestor_ip) */
  uint32_t flags;        /* YD_REQ_FLAG_* */
  int64_t expires_in_ns; /* lease length, counted from the grant */
} yd_task_req;

/* Outcome of one decision: flare::Expected<TaskAllocation, WaitStatus>
 * (task_dispatcher.h:69-77).  16 bytes. */
typedef struct yd_grant {
  uint64_t task_id;       /* valid iff status == YD_STATUS_GRANTED */
  uint32_t servant_index; /* registry position at grant time, else YD_NO_SERVANT */
  uint32_t status;        /* YD_STATUS_* */
} yd_grant;

/* RunningTask, yadcc/api/scheduler.proto:233-238. */
typedef struct yd_running_task {
  uint64_t servant_task_id;
  uint64_t task_grant_id;
  const char* servant_location;
  const char* task_digest;
} yd_running_task;

/* Per-servant bookkeeping exposed for parity checks; the same numbers the
 * reference publishes through DumpInternals (task_dispatcher.cc:548-584). */
typedef struct yd_servant_state {
  uint64_t running_tasks;       /* ServantDesc::running_tasks (h:189) */
  uint64_t ever_assigned_tasks; /* ServantDesc::ever_assigned_tasks (h:190) */
  uint64_t capacity_available;  /* GetCapacityAvailable (cc:283-313) */
  int64_t expires_at_ns;        /* ServantDesc::expires_at (h:187) */
} yd_servant_state;

/* Device-side timing of the most recent yd_wait_for_starting_new_tasks call
 * (CUDA backend; the oracles fill host wall-clock into solve_ms only). */
typedef struct yd_solve_stats {
  double total_ms;   /* H2D + all kernels + D2H, CUDA events on the solve stream */
  double solve_ms;   /* the assignment kernel alone */
  double prep_ms;    /* slot-table / classification kernels */
  double final_ms;   /* task-id scan + grant/lease write-out */
  uint64_t decisions;
  uint64_t granted;
  uint32_t kernel_launches; /* kernels launched by the call */
  uint32_t solver;          /* which solver ran (1 row-scan, 2 slot-stream) */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
} yd_solve_stats;

/* ---- lifecycle --------------------------------------------------------- */

/* TaskDispatcher::TaskDispatcher (cc:78-88).  Returns NULL if the config is
 * malformed or (CUDA backend) no usable sm_90 device is present -- the CUDA
 * backend never falls back to a CPU path. */
yd_sched* yd_create(const yd_config* cfg);
/* TaskDispatcher::~TaskDispatcher (cc:90-92). */
void yd_destroy(yd_sched* s);
/* "cuda-sm90a", "oracle-port" or "reference". */
const char* yd_backend_name(void);
/* yadcc::TryParseSize (yadcc/common/parse_size.cc:25-45).  Returns 1 and
 * stores the byte count on success, 0 when the reference returns nullopt. */
int yd_parse_size(const char* text, uint64_t* out_bytes);

/* ---- string interning (host only) --------------------------------------- */

/* Map a compiler digest / requestor IP string to a small id that yd_task_req
 * carries.  Ids are stable for the life of the handle.  yd_intern_ip returns
 * ids >= 1 (YD_IP_NONE is never returned, it is for callers that know the
 * requestor cannot be a servant). */
uint32_t yd_intern_env(yd_sched* s, const char* digest, size_t len);
uint32_t yd_intern_ip(yd_sched* s, const char* ip, size_t len);

/* ---- servant maintenance ------------------------------------------------ */

/* TaskDispatcher::KeepServantAlive (cc:190-220). */
void yd_keep_servant_alive(yd_sched* s, int64_t now_ns, const yd_servant* servant,
                           int64_t expires_in_ns);
/* TaskDispatcher::NotifyServantRunningTasks (cc:222-277).  Writes the unknown
 * task-grant ids (request order preserved) to unknown_out (capacity n) and
 * returns how many there are. */
size_t yd_notify_servant_running_tasks(yd_sched* s, const char* servant_location,
                                       const yd_running_task* tasks, size_t n,
                                       uint64_t* unknown_out);
/* One tick's worth of heartbeats in one call.  SchedulerServiceImpl::Heartbeat does KeepServantAlive
 * then NotifyServantRunningTasks per servant (scheduler_service_impl.cc:171-185); a scheduler front
 * end that collects the heartbeats of a tick issues them here as two batches.  Both calls are
 * defined as the loop over the single-servant calls above, in array order. */
typedef struct yd_heartbeat_item {
  const char* servant_location;  /* observed location, as for yd_notify_servant_running_tasks */
  const yd_running_task* tasks;  /* the servant's reported running tasks */
  size_t n_tasks;
} yd_heartbeat_item;
void yd_keep_servants_alive(yd_sched* s, int64_t now_ns, const yd_servant* servants,
                            const int64_t* expires_in_ns, size_t n);
/* unknown_out: the unknown ids of item 0, then item 1, ... (capacity: sum of n_tasks);
 * unknown_counts[i]: how many belong to item i.  Returns the total. */
size_t yd_notify_servants_running_tasks(yd_sched* s, const yd_heartbeat_item* items, size_t n,
                                        uint64_t* unknown_out, size_t* unknown_counts);
/* TaskDispatcher::GetRunningTasks (cc:279-281).  Returns the total count; at
 * most `cap` entries are written.  Returned strings are owned by the library
 * and valid until the next call that mutates the handle. */
size_t yd_get_running_tasks(yd_sched* s, yd_running_task* out, size_t cap);
/* TaskDispatcher::OnExpirationTimer (cc:498-536), fired by the caller at 1 Hz. */
void yd_on_expiration_timer(yd_sched* s, int64_t now_ns);

/* ---- task-grant allocation (THE HOT PATH) ------------------------------- */

/* n sequential TaskDispatcher::WaitForStartingNewTask calls (cc:93-140), in
 * array order, each with timeout == now (the zero-wait discipline
 * SchedulerServiceImpl itself uses for every request after the first,
 * scheduler_service_impl.cc:236-240).  out[i] is what call i would have
 * returned had the calls been issued one after another. */
void yd_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs,
                                    size_t n, yd_grant* out);

/* The same decisions over a narrower host<->device interface: 16 bytes up and 8 bytes down per
 * decision instead of 24 + 16 (PCIe is what an end-to-end batch of 100 k decisions spends most of
 * its time on).  Nothing is lost: the lease length is a count of milliseconds on the RPC surface
 * (scheduler.proto:197 WaitForStartingTaskRequest.next_keep_alive_in_ms; SchedulerServiceImpl multiplies
 * by 1ms, scheduler_service_impl.cc:221-222), and task ids are dense (next_task_id++ per grant,
 * task_dispatcher.cc:127), so the k-th grant of a batch has id first_task_id + k * stride. */
typedef struct yd_task_req16 {
  uint32_t env_id;       /* as yd_task_req */
  uint32_t min_version;
  uint32_t requestor_ip;
  uint32_t lease;        /* expires_in, milliseconds (< 2^31) | YD_LEASE_PREFETCH */
} yd_task_req16;
#define YD_LEASE_PREFETCH 0x80000000u

typedef struct yd_grant8 {
  uint32_t servant_index;  /* as yd_grant */
  uint32_t status_ordinal; /* YD_STATUS_* << 30 | FIFO ordinal of the grant inside the batch (0 unless granted) */
} yd_grant8;

typedef struct yd_packed_ids {
  uint64_t first_task_id; /* id of the batch's first grant */
  uint64_t stride;        /* 1 unless yd_config.id_stride says otherwise */
} yd_packed_ids;

static inline yd_task_req yd_unpack_req(yd_task_req16 r) {
  yd_task_req o;
  o.env_id = r.env_id;
  o.min_version = r.min_version;
  o.requestor_ip = r.requestor_ip;
  o.flags = (r.lease & YD_LEASE_PREFETCH) ? YD_REQ_FLAG_PREFETCH : 0u;
  o.expires_in_ns = (int64_t)(r.lease & 0x7fffffffu) * 1000000;
  return o;
}
static inline yd_grant yd_unpack_grant(yd_grant8 g, yd_packed_ids ids) {
  yd_grant o;
  o.status = g.status_ordinal >> 30;
  o.servant_index = g.servant_index;
  o.task_id = o.status == YD_STATUS_GRANTED ? ids.first_task_id + (uint64_t)(g.status_ordinal & 0x3fffffffu) * ids.stride : 0;
  return o;
}
static inline yd_grant8 yd_pack_grant(yd_grant g, yd_packed_ids ids) {
  yd_grant8 o;
  o.servant_index = g.servant_index;
  o.status_ordinal = (g.status << 30) |
                     (g.status == YD_STATUS_GRANTED ? (uint32_t)((g.task_id - ids.first_task_id) / ids.stride) : 0u);
  return o;
}

/* n decisions exactly as yd_wait_for_starting_new_tasks makes them.  *ids (may be NULL) receives what
 * turns ordinals into task ids; it is valid even if nothing was granted. */
void yd_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs,
                                           size_t n, yd_grant8* out, yd_packed_ids* ids);

/* The same call with the queue already in HBM.  A front end that receives requests over a
 * window of time can stage them as they arrive and start the solve when the batch closes:
 * yd_stage_requests copies reqs[0..n) into the handle's device-side queue (synchronously: the
 * array may be reused at once); yd_wait_for_staged_tasks decides the first n staged requests
 * exactly like yd_wait_for_starting_new_tasks would.  Staged requests stay valid, and may be
 * decided again, until the next call that replaces or drops them:
 *  - yd_stage_requests replaces them;
 *  - yd_wait_for_starting_new_tasks and yd_wait_for_starting_new_tasks_packed with n > 0 drop them
 *    (the batch goes through the same device-side queue);
 *  - yd_filter_and_wait_for_starting_new_tasks with n > 0 replaces them with the requests it
 *    offered, in order (none if every request was filtered out). */
void yd_stage_requests(yd_sched* s, const yd_task_req* reqs, size_t n);
void yd_wait_for_staged_tasks(yd_sched* s, int64_t now_ns, size_t n, yd_grant* out);
/* n TaskDispatcher::KeepTaskAlive calls (cc:142-165); ok_out[i] is the bool. */
void yd_keep_task_alive(yd_sched* s, int64_t now_ns, const uint64_t* task_ids, size_t n,
                        int64_t new_expires_in_ns, uint8_t* ok_out);
/* n TaskDispatcher::FreeTask calls (cc:167-188), one per id (so an unknown id
 * only skips itself, as in SchedulerServiceImpl::FreeTask, :307-309). */
void yd_free_tasks(yd_sched* s, const uint64_t* task_ids, size_t n);

/* ---- the caller's request expansion ---------------------------------------- */

/* Status codes of yadcc/api/scheduler.proto:23-35 that WaitForStartingTask can produce. */
#define YD_RPC_OK 0u
#define YD_RPC_NO_QUOTA_AVAILABLE 1001u
#define YD_RPC_INVALID_ARGUMENT 1004u
#define YD_RPC_ENVIRONMENT_NOT_AVAILABLE 1006u

/* One WaitForStartingTaskRequest (scheduler.proto:181-201) after token verification,
 * with the peer IP and the digest already interned. */
typedef struct yd_rpc_wait {
  uint32_t env_id;               /* env_desc.compiler_digest */
  uint32_t min_version;
  uint32_t requestor_ip;         /* EndpointGetIp(controller->GetRemotePeer()) */
  uint32_t immediate_reqs;
  uint32_t prefetch_reqs;
  uint32_t milliseconds_to_wait; /* only range-checked (<= 10 s); waiting is the caller's business */
  int64_t next_keep_alive_ns;    /* lease of every grant; must be <= 30 s */
} yd_rpc_wait;

typedef struct yd_rpc_wait_result {
  uint32_t status;      /* YD_RPC_* */
  uint32_t n_grants;    /* grants of this RPC ... */
  uint32_t first_grant; /* ... stored at grants_out[first_grant .. first_grant + n_grants) */
  uint32_t reserved;
} yd_rpc_wait_result;

/* n_rpcs SchedulerServiceImpl::WaitForStartingTask bodies (scheduler_service_impl.cc:
 * 209-271) executed back to back under the zero-wait discipline: each RPC expands to
 * `immediate_reqs` then `prefetch_reqs` sequential WaitForStartingNewTask calls with the
 * reference's stop rules (:234-264) and status mapping (:242-246, :266-270; note that an
 * unknown environment on a prefetch-only RPC yields NO_QUOTA, not ENVIRONMENT_NOT_AVAILABLE).
 * All RPCs are solved as ONE batch.  Returns the total number of grants written (<= cap;
 * cap must be >= yd_rpc_expanded_requests(), which is <= the sum of immediate_reqs + prefetch_reqs). */
size_t yd_wait_for_starting_task_rpcs(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs,
                                      yd_rpc_wait_result* results, yd_grant* grants_out, size_t cap);

/* Upper bound on the grants one batch can produce: sum over servants of min(num_processors,
 * max_tasks) (GetCapacityAvailable never exceeds either, task_dispatcher.cc:283-313). */
uint64_t yd_grant_capacity_bound(yd_sched* s);

/* Decisions yd_wait_for_starting_task_rpcs makes for these RPCs = the `cap` it needs.  Counts on
 * the wire are arbitrary uint32s; an RPC is expanded to at most yd_grant_capacity_bound() + 1
 * immediate and as many prefetch decisions, which is exact because nothing after an RPC's first
 * failed decision is reported (scheduler_service_impl.cc:247-251, :260-262).  The call returns
 * (size_t)-1, deciding nothing, if cap is too small, the batch exceeds 2^30 decisions or staging
 * memory cannot be had. */
size_t yd_rpc_expanded_requests(yd_sched* s, const yd_rpc_wait* rpcs, size_t n_rpcs);

/* ---- compilation-cache bloom pre-filter (SURVEY 8(f) row 1) ------------------- */

/* flare::experimental::SaltedBloomFilter (flare/base/experimental/bloom_filter.h:130,
 * :178-210, :249-305; hash = XXH64(s, len, 0), bloom_filter.cc:21-23): key k is tested /
 * added through num_hashes probes h_i = XXH64(le32(i) || key), bit = h_i & (bits - 1),
 * stored as bytes[bit / 8] & (1 << bit % 8).  yadcc's cache server builds it with
 * 27 584 639 -> 2^25 bits and 10 hashes (yadcc/cache/bloom_filter_generator.h:65-68) and the
 * delegate daemon consults it before asking the scheduler for a grant
 * (yadcc/daemon/local/distributed_cache_reader.cc:70-77).  One filter per handle.
 *
 * Keys are passed as n fixed-length records: key i = keys + i * stride, key_len bytes. */

/* BloomFilter(m, k): empty filter of max(8, next_pow2(m)) bits.  Returns 0 on success. */
int yd_bloom_reset(yd_sched* s, uint64_t size_in_bits, uint32_t num_hashes);
/* BloomFilter(existing_filter, k): n_bytes * 8 must be a power of two. */
int yd_bloom_load(yd_sched* s, const uint8_t* bytes, size_t n_bytes, uint32_t num_hashes);
/* BloomFilter::Add for n keys. */
void yd_bloom_add(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride);
/* BloomFilter::PossiblyContains for n keys; out[i] = 0 / 1. */
void yd_bloom_possibly_contains(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride,
                                uint8_t* out);
/* BloomFilter::GetBytes: returns the filter size in bytes; copies at most cap bytes. */
size_t yd_bloom_get_bytes(yd_sched* s, uint8_t* out, size_t cap);

/* ---- in-flight task index (SURVEY 8(f) row 2) ------------------------------ */

/* The delegate daemon's RunningTaskKeeper (yadcc/daemon/local/running_task_keeper.cc:40-75):
 * once a second it replaces its map  task_digest -> {servant_location, servant_task_id}  with the
 * scheduler's GetRunningTasks answer (a later entry with the same digest overwrites an earlier
 * one, cc:56-60) and, before asking for a grant, looks the new task's digest up
 * (TryFindTask, cc:67-75; caller distributed_task_dispatcher.cc:257) so that a translation
 * unit already being compiled somewhere is joined instead of compiled twice.  Here the map is
 * built from the handle's own running-task bookkeeping and probed for a whole queue at once. */
typedef struct yd_running_hit {
  uint64_t servant_task_id; /* TaskDesc::servant_task_id (running_task_keeper.h:39), 0 if not found */
  uint32_t snapshot_index;  /* position of the winning entry in the refreshed snapshot (the order
                             * yd_get_running_tasks returned at refresh time), YD_NO_SERVANT if not found */
  uint32_t found;           /* TryFindTask(...).has_value() */
} yd_running_hit;

/* RunningTaskKeeper::Refresh (cc:40-65) against this handle: snapshot = what
 * yd_get_running_tasks returns now.  Returns the number of entries in the snapshot. */
size_t yd_running_index_refresh(yd_sched* s);
/* Number of distinct digests in the index (running_tasks_.size()). */
size_t yd_running_index_size(yd_sched* s);
/* TryFindTask x n.  Keys are n fixed-length records like the bloom calls:
 * key i = keys + i * stride, key_len bytes. */
void yd_running_index_find(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride,
                           yd_running_hit* out);
/* Entry `snapshot_index` of the refreshed snapshot; returns 0 if out of range.  The strings
 * stay valid until the next yd_running_index_refresh. */
int yd_running_index_entry(yd_sched* s, uint32_t snapshot_index, yd_running_task* out);

/* ---- BASELINE configs[3] as one call: pre-filters + solve ------------------------------- */

/* What a delegate daemon does for every task before a grant is asked, for a whole queue at once:
 * (1) the compilation cache's bloom filter (yd_bloom_possibly_contains; a possible hit is served
 * from the cache, distributed_cache_reader.cc:70-77), (2) the in-flight task index
 * (yd_running_index_find; an identical task already running is joined,
 * distributed_task_dispatcher.cc:257) and (3) yd_wait_for_starting_new_tasks over what is left,
 * FIFO order kept.  Either filter stage is skipped when its key array is NULL. */
typedef struct yd_prefilter {
  const char* cache_keys; /* n fixed-length records like the bloom calls, or NULL */
  size_t cache_key_len, cache_key_stride;
  const char* task_digests; /* n fixed-length records like yd_running_index_find, or NULL */
  size_t task_digest_len, task_digest_stride;
} yd_prefilter;
#define YD_FILTER_OFFERED 0u   /* went to the scheduler: its grant is the next unread entry of grants_out */
#define YD_FILTER_CACHE_HIT 1u /* BloomFilter::PossiblyContains(cache key) */
#define YD_FILTER_JOINED 2u    /* TryFindTask(task digest).has_value(), and no cache hit */
/* verdict_out[i] (n bytes) = YD_FILTER_*; hits_out (n entries, may be NULL) = what
 * yd_running_index_find reports for request i; grants_out (capacity n): the decisions for the
 * OFFERED requests, in order.  Returns how many requests were offered.  Defined as the three calls
 * above applied in that order, the third as yd_stage_requests(offered) + yd_wait_for_staged_tasks:
 * the offered requests stay staged afterwards.  The CUDA backend keeps the queue in HBM between the
 * stages. */
size_t yd_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n,
                                                 const yd_prefilter* filter, uint8_t* verdict_out,
                                                 yd_running_hit* hits_out, yd_grant* grants_out);

/* ---- introspection ------------------------------------------------------ */

size_t yd_num_servants(yd_sched* s);
/* observed_location of registry position `servant_index`; NULL if out of
 * range.  Valid until the next mutating call. */
const char* yd_servant_location(yd_sched* s, uint32_t servant_index);
/* Fills up to `cap` entries in registry order; returns the servant count. */
size_t yd_get_servant_state(yd_sched* s, yd_servant_state* out, size_t cap);
/* ServantPersonality of registry position `servant_index` as last reported (h:80-116).
 * Strings and the digest array stay valid until the next call on the handle.  Returns 0 if
 * out of range. */
int yd_get_servant_personality(yd_sched* s, uint32_t servant_index, yd_servant* out);
/* Next task id that would be handed out (TaskRegistry::next_task_id, h:218). */
uint64_t yd_next_task_id(yd_sched* s);
/* Number of live (granted, not freed/swept) task leases, zombies included. */
uint64_t yd_num_tasks(yd_sched* s);
/* DumpInternals summary (cc:538-614) as JSON: servants_up, running_tasks,
 * capacity, capacity_available, capacity_unavailable.  Returns the length
 * needed (excluding NUL); writes at most cap bytes. */
size_t yd_dump_internals_json(yd_sched* s, char* buf, size_t cap);
/* Returns 1 and fills *out if a solve has run on this handle. */
int yd_last_solve_stats(yd_sched* s, yd_solve_stats* out);

/* ---- host staging buffers ----------------------------------------------- */

/* Page-locked host memory for request / grant arrays, so that the copies in
 * yd_wait_for_starting_new_tasks are single DMA transfers.  The CPU oracles
 * implement these with malloc/free. */
void* yd_alloc_host(size_t bytes);
void yd_free_host(void* p);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* YDSCHED_H_ */
