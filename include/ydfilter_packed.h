/* ydfilter_packed.h -- the pre-filtered solve (yd_filter_and_wait_for_starting_new_tasks, ydsched.h) over the packed
 * interface: the requests as yd_task_req16, the cache keys and task digests as the 32-byte binary digests they are the
 * hex of, the grants as yd_grant8.  Exported by the CUDA library; the CPU checkers export it from builds of their own
 * (include/ydsched_filter_packed_impl.inc).  The range-sharded group's form is in ydshard.h. */
#ifndef YDFILTER_PACKED_H_
#define YDFILTER_PACKED_H_

#include "ydsched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The pre-filters of yd_filter_and_wait_for_starting_new_tasks over binary digests: n contiguous 32-byte records each,
 * or NULL to skip that stage.  Record i stands for the key the delegate derives from it (yadcc/cache/cache_format.cc:
 * 56-64, yadcc/daemon/local/task_digest.cc:25-30):
 *   cache key   = "yadcc-cxx2-entry-" + lowercase hex(cache_digests[i])   (81 bytes)
 *   task digest = lowercase hex(task_digests[i])                          (64 bytes)
 * 16 bytes. */
typedef struct yd_prefilter_packed {
  const uint8_t* cache_digests;
  const uint8_t* task_digests;
} yd_prefilter_packed;

/* yd_filter_and_wait_for_starting_new_tasks over the packed interface: 16 + 32 + 32 bytes up per request instead of
 * 24 + 81 + 64, and 8 bytes down per offered request instead of 16.  Defined as that call on yd_unpack_req(reqs[i])
 * with the hex-expanded keys, then yd_pack_grant of each grant with the batch's *ids (may be NULL; valid even if
 * nothing was offered): verdicts, hits, FIFO order and staging afterwards (the offered requests, as 24-byte records)
 * are that call's. */
size_t yd_filter_and_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs, size_t n,
                                                        const yd_prefilter_packed* filter, uint8_t* verdict_out,
                                                        yd_running_hit* hits_out, yd_grant8* grants_out,
                                                        yd_packed_ids* ids);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* YDFILTER_PACKED_H_ */
