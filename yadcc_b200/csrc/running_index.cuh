// running_index.cuh -- the in-flight task index (SURVEY 8(f) row 2).
//
// RunningTaskKeeper (yadcc/daemon/local/running_task_keeper.cc:40-75) keeps
// unordered_map<task_digest, {servant_location, servant_task_id}>, rebuilt every second from the
// scheduler's GetRunningTasks answer with `tmp[digest] = desc` (a later entry of the same digest
// wins, cc:56-60), and TryFindTask probes it once per new compilation task.  Here the map
// is an open-addressing table in HBM whose slots hold (snapshot index + 1): building it is
// one pass over the snapshot (atomicCAS to claim a slot, atomicMax so the LAST entry of a
// digest wins, whatever the thread order), and a whole pending queue is probed in one launch.
// Results do not depend on the hash function -- only on key equality -- so it is a private
// 64-bit mix, not XXH64.
//
// Algorithmic bytes: build reads each stored digest once (+4 B slot); find reads each
// query key once, the slot(s) it probes (4 B) and the candidate digest (key_len B), and writes
// a 16-byte verdict.
#pragma once
#include "common.cuh"

namespace yd {

struct RtIndex {
  const unsigned char* bytes;  // stored digests, each starting on an 8-byte boundary
  const uint32_t* off;         // [n] byte offset of entry i
  const uint32_t* len;         // [n] its length
  uint32_t* slots;             // [mask + 1] 0 = empty, else snapshot index + 1
  uint32_t mask;
};

// Little-endian 8-byte word `w` of a key of `len` bytes, zero padded.
__device__ __forceinline__ unsigned long long rt_word(const unsigned char* p, uint32_t len, uint32_t w) {
  const uint32_t b0 = w * 8;
  if (b0 + 8 <= len && ((reinterpret_cast<uintptr_t>(p) & 7u) == 0)) {
    return *reinterpret_cast<const unsigned long long*>(p + b0);
  }
  unsigned long long v = 0;
  for (uint32_t k = 0; k < 8 && b0 + k < len; ++k) v |= (unsigned long long)p[b0 + k] << (8 * k);
  return v;
}

// A key as the index hashes and compares it: len bytes, read as little-endian 8-byte words, zero padded.
// Fixed-length records and stored digests: bytes in memory.
struct RtBytes {
  const unsigned char* p;
  uint32_t len;
  __device__ __forceinline__ unsigned long long word(uint32_t w) const { return rt_word(p, len, w); }
};
// A 32-byte binary task digest (yd_prefilter_packed) as the 64-character lowercase hex it stands for, in registers.
struct RtHex {
  static constexpr uint32_t len = 64;
  unsigned long long h[8];
  __device__ __forceinline__ unsigned long long word(uint32_t w) const { return h[w]; }
};

template <class K>
__device__ __forceinline__ unsigned long long rt_hash(const K& k) {
  unsigned long long h = 0x9E3779B97F4A7C15ull ^ k.len;
  for (uint32_t w = 0; w * 8 < k.len; ++w) {
    h ^= k.word(w);
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 32;
  }
  h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 29;
  return h;
}

template <class K>
__device__ __forceinline__ bool rt_equal(const K& a, const RtBytes& b) {
  if (a.len != b.len) return false;
  for (uint32_t w = 0; w * 8 < a.len; ++w) {
    if (a.word(w) != b.word(w)) return false;
  }
  return true;
}

// Query loaders of k_rt_find: key(q) is query q.
// Fixed-length records: query q = keys + q * stride, key_len bytes.
struct RtRecords {
  const unsigned char* keys;
  size_t stride;
  uint32_t key_len;
  __device__ __forceinline__ RtBytes key(uint32_t q) const { return RtBytes{keys + (size_t)q * stride, key_len}; }
};
// 32-byte task digests: query q = lowercase hex(digests + 32 q).  A stored digest that is not 64 bytes of lowercase hex
// never matches.
struct RtTaskDigests {
  const unsigned char* digests;
  __device__ __forceinline__ RtHex key(uint32_t q) const {
    RtHex k;
    hex_digest(digests + (size_t)q * 32, k.h);
    return k;
  }
};

// One thread per snapshot entry.
__global__ void __launch_bounds__(256) k_rt_build(RtIndex ix, uint32_t n, uint32_t* __restrict__ distinct) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const RtBytes key{ix.bytes + ix.off[i], ix.len[i]};
  uint32_t h = (uint32_t)rt_hash(key) & ix.mask;
  for (uint32_t probe = 0; probe <= ix.mask; ++probe) {
    uint32_t cur = ix.slots[h];
    if (cur == 0) {
      cur = atomicCAS(&ix.slots[h], 0u, i + 1);
      if (cur == 0) { atomicAdd(distinct, 1u); return; }  // claimed an empty slot: a new digest
    }
    // the slot belongs to some digest for good (only its entry index can grow): is it mine?
    const uint32_t o = cur - 1;
    if (rt_equal(key, RtBytes{ix.bytes + ix.off[o], ix.len[o]})) {
      atomicMax(&ix.slots[h], i + 1);  // tmp[digest] = desc: the last entry wins (cc:59)
      return;
    }
    h = (h + 1) & ix.mask;
  }
}

// One thread per query key.
template <class Keys>
__global__ void __launch_bounds__(256) k_rt_find(RtIndex ix, Keys keys, uint32_t n,
                                                 const unsigned long long* __restrict__ servant_task_id,
                                                 uint4* __restrict__ out /* yd_running_hit */) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  uint4 verdict = make_uint4(0u, 0u, kNone, 0u);
  if (ix.slots != nullptr) {
    const auto key = keys.key(q);
    uint32_t h = (uint32_t)rt_hash(key) & ix.mask;
    for (uint32_t probe = 0; probe <= ix.mask; ++probe) {
      const uint32_t cur = ix.slots[h];
      if (cur == 0) break;
      const uint32_t o = cur - 1;
      if (rt_equal(key, RtBytes{ix.bytes + ix.off[o], ix.len[o]})) {
        const unsigned long long id = servant_task_id[o];
        verdict = make_uint4((uint32_t)id, (uint32_t)(id >> 32), o, 1u);
        break;
      }
      h = (h + 1) & ix.mask;
    }
  }
  out[q] = verdict;
}

}  // namespace yd
