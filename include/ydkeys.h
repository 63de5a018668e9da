/* ydkeys.h -- the delegate's cache keys and task digests derived from task descriptors, and the pre-filtered solve
 * (yd_filter_and_wait_for_starting_new_tasks, ydsched.h) started from those descriptors.  Exported by the CUDA library;
 * the CPU checkers export it from builds of their own. */
#ifndef YDKEYS_H_
#define YDKEYS_H_

#include "ydsched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- the same queue from task descriptors: cache keys and task digests derived here ------------ */

/* A delegate daemon derives both filter keys from the task it holds (cxx_compilation_task.cc:40,44):
 *   cache key   = "yadcc-cxx2-entry-" + hex(BLAKE3("using-extra-info" || compiler_digest || args || source_digest))
 *                 (GetCxxCacheEntryKey, yadcc/daemon/cache_format.cc:56-64), 81 bytes;
 *   task digest = hex(BLAKE3("cxx2" || compiler_digest || args || source_digest))
 *                 (GetCxxTaskDigest, yadcc/daemon/task_digest.cc:25-30), 64 bytes;
 * hex in lower case, compiler_digest = the string yd_intern_env mapped to the request's env_id.  The
 * invocation-argument strings are few and long, so a call passes each distinct one once and every request
 * names its string by index.  Nothing of this is kept by the handle after the call. */
typedef struct yd_task_sources {
  const char* args;              /* the call's distinct invocation-argument strings, back to back (any bytes) */
  const uint64_t* args_offsets;  /* n_args + 1 non-decreasing offsets into args: string k = [off[k], off[k+1]) */
  size_t n_args;
  const uint32_t* args_index;    /* per request: which string, < n_args */
  const char* source_digests;    /* per request: record i = source_digests + i * stride, source_digest_len bytes */
  size_t source_digest_len, source_digest_stride;
} yd_task_sources;

#define YD_KEYS_OK 0
#define YD_KEYS_BAD_SOURCES 1    /* args_offsets not non-decreasing from 0, or a NULL array that is needed */
#define YD_KEYS_UNKNOWN_ENV 2    /* a request's env_id was never interned */
#define YD_KEYS_BAD_ARGS_INDEX 3 /* a request's args_index >= n_args */
#define YD_KEYS_TOO_LONG 4       /* a string above its limit: see below */
#define YD_KEYS_CACHE_KEY_LEN 81
#define YD_KEYS_TASK_DIGEST_LEN 64
/* Longest invocation-argument string a call takes (256 KiB; BLAKE3 hashes messages past 1024 bytes as
 * a tree of chunks), and longest compiler digest (of a request's env_id) and source digest (64 KiB). */
#define YD_KEYS_MAX_ARGS_LEN (256u << 10)
#define YD_KEYS_MAX_DIGEST_LEN (64u << 10)

/* GetCxxCacheEntryKey / GetCxxTaskDigest for n requests.  cache_keys_out: n x 81 bytes,
 * task_digests_out: n x 64 bytes; either may be NULL.  Returns YD_KEYS_OK, or the YD_KEYS_* error of the
 * first failing check with nothing written: the sources are checked first (offsets, then every string's
 * length and source_digest_len), then the requests in order (env_id, then the compiler digest's length,
 * then args_index). */
int yd_derive_task_keys(yd_sched* s, const yd_task_req* reqs, size_t n, const yd_task_sources* src,
                        char* cache_keys_out, char* task_digests_out);

#define YD_STAGE_CACHE 1u  /* probe the bloom filter with the derived cache keys */
#define YD_STAGE_DEDUPE 2u /* probe the in-flight index with the derived task digests */
/* Defined as yd_derive_task_keys, then yd_filter_and_wait_for_starting_new_tasks with the derived records
 * (stride 81 / 64) for the stages selected in `stages`.  Same outputs, same "offered requests stay staged"
 * rule.  Returns (size_t)-1 and decides nothing (the staged queue is kept) on a YD_KEYS_* error.  The CUDA
 * backend derives the keys on the device, straight into the buffers the filter stages read, so only the
 * descriptors are uploaded. */
size_t yd_derive_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n,
                                                        const yd_task_sources* src, uint32_t stages,
                                                        uint8_t* verdict_out, yd_running_hit* hits_out,
                                                        yd_grant* grants_out);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* YDKEYS_H_ */
