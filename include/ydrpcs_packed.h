/* ydrpcs_packed.h -- a window of WaitForStartingTask RPCs (yd_wait_for_starting_task_rpcs, ydsched.h) with 8-byte grants
 * (yd_grant8) down.  Exported by the CUDA library, which expands the window, applies the stop rules and the status
 * mapping on the device; the CPU checkers export it from builds of their own (include/ydsched_rpc_packed_impl.inc).  The
 * range-sharded group's form is in ydshard.h. */
#ifndef YDRPCS_PACKED_H_
#define YDRPCS_PACKED_H_

#include "ydsched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* yd_wait_for_starting_task_rpcs on the same arguments, then yd_pack_grant of every grant with the window's *ids
 * = {next task id before the call, stride} (ids may be NULL; *ids is valid even if nothing was granted).  Results,
 * refusals ((size_t)-1, nothing decided: cap < yd_rpc_expanded_requests(), more than 2^30 decisions, no staging memory)
 * and the state afterwards (servants, leases, next task id, the staged queue) are that call's.  The RPC records are the
 * 32-byte yd_rpc_wait, next_keep_alive_ns carried exactly; 16 bytes per RPC and 8 per grant come back.
 *
 * The ordinal of grants_out[k] is k: every granted decision of the window is reported.  All decisions of one RPC share
 * class and requestor, failed decisions change no state, and within a batch running_tasks only grows, so a class that
 * failed once keeps failing: a granted decision never follows a failed one of its own RPC.  So the task id of
 * grants_out[k] is ids->first_task_id + k * ids->stride. */
size_t yd_wait_for_starting_task_rpcs_packed(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs,
                                             yd_rpc_wait_result* results, yd_grant8* grants_out, size_t cap,
                                             yd_packed_ids* ids);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* YDRPCS_PACKED_H_ */
