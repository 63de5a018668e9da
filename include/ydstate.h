/*
 * ydstate.h -- export and import of a scheduler handle's decision state.
 *
 * A scheduler process that restarts (library upgrade, a move to another GPU, recovery after a crash)
 * loses every lease it granted: at their next heartbeat the servants report their running tasks, the
 * fresh handle knows none of them and NotifyServantRunningTasks tells the servants to kill them
 * (task_dispatcher.cc:256-273), and task ids start again at 0.  Exporting the state before the old
 * process ends and importing it into the new handle keeps servants, leases and task ids: the imported
 * handle makes the same decisions, call after call, as the handle that never stopped.
 *
 * Exported: the servant registry, the lease map, next_task_id, the running-task bookkeeper and both
 * intern tables.  Not exported (the imported handle starts with these cold, like a fresh one): the
 * staged request queue, the bloom filter (it has yd_bloom_get_bytes / yd_bloom_load of its own), the
 * in-flight task index (rebuilt by the next yd_running_index_refresh), solve statistics, caches, and
 * everything of the service layer (include/ydservice.h).
 *
 * TIME.  Every absolute time in the export is stored relative to the export's `now_ns` and rebased
 * onto the import's `now_ns`: time stands still while the state is in transit.  No daemon could renew
 * a lease and no servant could heartbeat while no scheduler ran, so the downtime must not count
 * against them.  It also means the exporting and the importing process need no common clock origin.
 *
 * FORMAT, version 1.  Little-endian, no padding, no alignment.  str = u32 byte length + bytes.
 *
 *   header      u32 magic 0x54534459 ("YDST")   u32 version (1)
 *               u32 id_stride (1 when the config says 0)   u32 id_offset
 *               u64 servant_min_memory_for_accepting_new_task, parsed, in bytes
 *               u64 next_task_id (the id the next grant gets, yd_next_task_id)
 *   envs        u32 count, then `count` str: yd_intern_env's table in id order
 *   ips         u32 count, then `count` str: yd_intern_ip's table in id order (id 0 is "")
 *   servants    u32 count, then per servant in registry order:
 *                 i32 version  i32 priority  i32 not_accepting_task_reason
 *                 u32 num_processors  u32 current_load  u32 max_tasks
 *                 u64 total_memory_in_bytes  u64 memory_available_in_bytes
 *                 i64 expires_at - now  u64 ever_assigned_tasks
 *                 str observed_location  str reported_location
 *                 u32 num_envs, then num_envs str: the environment digests in heartbeat order
 *               (running_tasks is not stored: it always equals the number of leases on the servant,
 *               zombies included, and the import counts them)
 *   leases      u64 count, then per lease in ascending id order, 24 bytes:
 *                 u64 task id   u32 servant registry position
 *                 u32 flags (YD_STATE_LEASE_*)   i64 expires_at - now
 *   bookkeeper  u64 bucket_count of RunningTaskBookkeeper's unordered_map
 *               u32 groups, then per group in the map's iteration order:
 *                 str servant location   u32 tasks, then per task:
 *                 u64 servant_task_id  u64 task_grant_id  str servant_location  str task_digest
 *
 * The export is canonical: backends fed the same calls produce the same bytes, with one caveat on the
 * intern tables.  The CUDA backend also interns the digests servants report and the IPs of servant
 * locations (they index its device-side topology), the CPU backends do not, so the tables of two
 * backends agree only when the caller has interned those strings itself before the handle did.
 *
 * The bookkeeper's iteration order is observable (GetRunningTasks; the in-flight index's "later entry
 * wins", running_task_keeper.cc:56-60) and depends on the map's history.  Import reproduces it by
 * rehashing the empty map to the stored bucket count (unless that count is 1: a never-used map) and
 * inserting the groups in reverse iteration order.
 */
#ifndef YDSTATE_H_
#define YDSTATE_H_

#include <stddef.h>
#include <stdint.h>

#include "ydsched.h"

#ifdef __cplusplus
extern "C" {
#endif

#define YD_STATE_MAGIC 0x54534459u
#define YD_STATE_VERSION 1u

#define YD_STATE_LEASE_PREFETCH 1u /* TaskDesc::is_prefetch */
#define YD_STATE_LEASE_ZOMBIE 2u   /* TaskDesc::zombie */

#define YD_STATE_OK 0
#define YD_STATE_BAD_BLOB 1         /* truncated, wrong magic / version, inconsistent contents, or a live
                                     * window (oldest lease to next_task_id) wider than 2^40 ids */
#define YD_STATE_NOT_FRESH 2        /* the target handle has seen calls other than yd_create */
#define YD_STATE_CONFIG_MISMATCH 3  /* id_stride, id_offset or the minimum memory differ from the export's */
#define YD_STATE_UNSUPPORTED 4      /* the handle joined a range-sharded queue: yd_shard_import_state (ydshard.h) */
#define YD_STATE_NO_MEMORY 5        /* a valid export whose lease window does not fit the device's free memory
                                     * now (CUDA backend); the export is fine, retry when there is room */

/* Serialise the handle's decision state.  Returns the byte count; writes the export to out only if
 * cap suffices (out may be NULL with cap 0 to ask for the size).  Returns 0 if the backend cannot
 * export the handle: a range-sharded handle holds only its own leases, and its group exports together
 * with yd_shard_export_state (ydshard.h).  Decisions after an export are those the handle would have
 * made without it. */
size_t yd_export_state(yd_sched* s, int64_t now_ns, uint8_t* out, size_t cap);

/* Load an export into a FRESH handle (yd_create, then nothing but this call).  Returns YD_STATE_*.
 * Every refusal (malformed input: YD_STATE_BAD_BLOB) leaves the handle fresh. */
int yd_import_state(yd_sched* s, int64_t now_ns, const uint8_t* blob, size_t len);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* YDSTATE_H_ */
