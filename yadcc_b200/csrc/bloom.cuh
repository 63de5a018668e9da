// bloom.cuh -- the compilation-cache bloom pre-filter on the GPU (SURVEY 8(f) row 1).
//
// flare::experimental::SaltedBloomFilter (flare/base/experimental/bloom_filter.h:130,
// :178-210, :249-305): key k is probed with h_i = XXH64(le32(i) || k, seed 0) for
// i = 0 .. num_hashes-1 (bloom_filter.cc:21-23), bit = h_i & (bits - 1), stored as
// bytes[bit / 8] & (1 << bit % 8).  yadcc: 2^25 bits, 10 hashes
// (yadcc/cache/bloom_filter_generator.h:65-68); the 4 MiB table stays L2-resident.
//
// One thread per key.  The key is pulled into registers once (fixed key length per call,
// 8-byte words), and the 10 salted hashes reuse it: only the first 8-byte lane of the
// first stripe depends on the salt.  XXH64 is written out from the published xxHash
// specification.  Algorithmic bytes: key_len per key read + num_hashes random 1-byte
// probes (Add: atomicOr on 4-byte words).
#pragma once
#include "common.cuh"

namespace yd {

constexpr unsigned long long kXP1 = 11400714785074694791ull, kXP2 = 14029467366897019727ull,
                             kXP3 = 1609587929392839161ull, kXP4 = 9650029242287828579ull,
                             kXP5 = 2870177450012600261ull;
constexpr int kBloomMaxKey = 252;  // salted buffer <= 256 bytes lives in registers / local memory

__device__ __forceinline__ unsigned long long xrotl(unsigned long long x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ unsigned long long xround(unsigned long long acc, unsigned long long in) {
  return xrotl(acc + in * kXP2, 31) * kXP1;
}
__device__ __forceinline__ unsigned long long xmerge(unsigned long long h, unsigned long long v) {
  return (h ^ xround(0, v)) * kXP1 + kXP4;
}

// XXH64 over a buffer held as little-endian 8-byte words (w[i] = bytes 8i .. 8i+7).
__device__ __forceinline__ unsigned long long xxh64_words(const unsigned long long* w, uint32_t len) {
  uint32_t pos = 0;  // in bytes, always a multiple of 8 while whole words remain
  unsigned long long h;
  if (len >= 32) {
    unsigned long long v1 = kXP1 + kXP2, v2 = kXP2, v3 = 0, v4 = 0ull - kXP1;
    do {
      const uint32_t i = pos >> 3;
      v1 = xround(v1, w[i]); v2 = xround(v2, w[i + 1]); v3 = xround(v3, w[i + 2]); v4 = xround(v4, w[i + 3]);
      pos += 32;
    } while (pos + 32 <= len);
    h = xrotl(v1, 1) + xrotl(v2, 7) + xrotl(v3, 12) + xrotl(v4, 18);
    h = xmerge(h, v1); h = xmerge(h, v2); h = xmerge(h, v3); h = xmerge(h, v4);
  } else {
    h = kXP5;
  }
  h += len;
  while (pos + 8 <= len) { h = xrotl(h ^ xround(0, w[pos >> 3]), 27) * kXP1 + kXP4; pos += 8; }
  unsigned long long tail = pos < len ? w[pos >> 3] : 0;  // up to 7 remaining bytes
  if (pos + 4 <= len) { h = xrotl(h ^ ((tail & 0xffffffffull) * kXP1), 23) * kXP2 + kXP3; pos += 4; tail >>= 32; }
  while (pos < len) { h = xrotl(h ^ ((tail & 0xffull) * kXP5), 11) * kXP1; ++pos; tail >>= 8; }
  h ^= h >> 33; h *= kXP2; h ^= h >> 29; h *= kXP3; h ^= h >> 32;
  return h;
}

// Key loaders of k_bloom: load(i, w) writes key i into the salted buffer w from byte 4 on (the salt's 4 bytes are
// rewritten per probe) and returns the buffer's length.

// Fixed-length records: key i = keys + i * stride, key_len bytes.
struct BloomRecords {
  static constexpr int kWords = (kBloomMaxKey + 4 + 7) / 8;
  const unsigned char* keys;
  size_t stride;
  uint32_t key_len;
  __device__ __forceinline__ uint32_t load(uint32_t i, unsigned long long* w) const {
    const unsigned char* k = keys + (size_t)i * stride;
    const uint32_t total = key_len + 4;
    const uint32_t nwords = (total + 7) / 8;
    for (uint32_t j = 0; j < nwords; ++j) {
      unsigned long long v = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        const uint32_t at = j * 8 + b;  // byte of the salted buffer
        if (at >= 4 && at < total) v |= (unsigned long long)k[at - 4] << (8 * b);
      }
      w[j] = v;
    }
    return total;
  }
};

// 32-byte cache digests (yd_prefilter_packed): key i = "yadcc-cxx2-entry-" + lowercase hex(digests + 32 i), 81 bytes.
// The salted buffer is 85 bytes: salt, the prefix at bytes 4 .. 20, the hex at 21 .. 84, i.e. hex word k (characters
// 8k .. 8k+7) straddles buffer words k + 2 (its first 3 characters, at bytes 5 .. 7) and k + 3 (the other 5).
struct BloomCacheDigests {
  static constexpr int kWords = 11;
  const unsigned char* digests;
  __device__ __forceinline__ uint32_t load(uint32_t i, unsigned long long* w) const {
    unsigned long long h[8];
    hex_digest(digests + (size_t)i * 32, h);
    w[0] = 0x6364617900000000ull;  // salt | "yadc"
    w[1] = 0x652d327878632d63ull;  // "c-cxx2-e"
    w[2] = 0x0000002d7972746eull | (h[0] << 40);  // "ntry-"
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k + 3] = (h[k] >> 24) | (k < 7 ? h[k + 1] << 40 : 0ull);
    return 85;
  }
};

// kAdd = false: PossiblyContains -> out[i]; kAdd = true: Add (atomicOr into the table).
template <bool kAdd, class Keys>
__global__ void __launch_bounds__(128) k_bloom(Keys keys, uint32_t n, uint32_t num_hashes, unsigned long long mask,
                                               uint32_t* __restrict__ table /* bytes viewed as le32 words */,
                                               uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // salted buffer: 4 bytes of salt, then the key
  unsigned long long w[Keys::kWords];
  const uint32_t total = keys.load(i, w);
  bool all = true;
  for (uint32_t salt = 0; salt < num_hashes; ++salt) {
    w[0] = (w[0] & 0xffffffff00000000ull) | salt;  // SaltInteger = int, little endian (:181,:201-203)
    const unsigned long long bit = xxh64_words(w, total) & mask;
    const uint32_t word = (uint32_t)(bit >> 5), m = 1u << (bit & 31);  // byte bit/8, bit%8 == le32 word bit/32, bit%32
    if (kAdd) {
      atomicOr(&table[word], m);
    } else if (!(table[word] & m)) {
      all = false;
      break;  // PossiblyContains stops at the first clear bit (:256-261)
    }
  }
  if (!kAdd) out[i] = all ? 1 : 0;
}

}  // namespace yd
