// ref_keys.cc -- TEST INFRASTRUCTURE: the reference harness (ref_harness.cc) plus the task keys of a delegate
// (yd_derive_task_keys, yd_derive_filter_and_wait_for_starting_new_tasks) over flare's own Blake3 and EncodeHex and the
// vendored BLAKE3 C, compiled verbatim by oracle/keys.mk into _ref/libydref_keys.so.
#include "ref_harness.cc"
#include "ydsched_keys_impl.inc"

// ---- task keys: flare's own Blake3 over the vendored BLAKE3 C, flare's EncodeHex ------------------------------
// cache_format.cc pulls in protobuf, so GetCxxCacheEntryKey (cache_format.cc:56-64) and GetCxxTaskDigest
// (task_digest.cc:25-30) are restated here, their formula lines as they stand.
#include "flare/base/crypto/blake3.h"
#include "flare/base/encoding/hex.h"

extern "C" int yd_derive_task_keys(yd_sched* s, const yd_task_req* reqs, size_t n, const yd_task_sources* src,
                                   char* cache_keys_out, char* task_digests_out) {
  if (int rc = yd_keys_check(s->envs, reqs, n, src)) return rc;
  for (size_t i = 0; i != n; ++i) {
    const std::string_view compiler_digest = s->envs[reqs[i].env_id];
    const uint32_t a = src->args_index[i];
    const std::string_view invocation_arguments(src->args + src->args_offsets[a], src->args_offsets[a + 1] - src->args_offsets[a]);
    const std::string_view source_digest(src->source_digests + i * src->source_digest_stride, src->source_digest_len);
    if (cache_keys_out) {
      const std::string key = "yadcc-cxx2-entry-" + flare::EncodeHex(flare::Blake3(
                                                        {"using-extra-info", compiler_digest, invocation_arguments, source_digest}));
      std::memcpy(cache_keys_out + i * YD_KEYS_CACHE_KEY_LEN, key.data(), YD_KEYS_CACHE_KEY_LEN);
    }
    if (task_digests_out) {
      const std::string digest = flare::EncodeHex(flare::Blake3({"cxx2", compiler_digest, invocation_arguments, source_digest}));
      std::memcpy(task_digests_out + i * YD_KEYS_TASK_DIGEST_LEN, digest.data(), YD_KEYS_TASK_DIGEST_LEN);
    }
  }
  return YD_KEYS_OK;
}

#include "ydsched_derive_impl.inc"
