// blake3.cuh -- the delegate's cache keys and task digests, derived on the device from task descriptors.
//
//   cache key   = "yadcc-cxx2-entry-" + hex(BLAKE3("using-extra-info" || compiler_digest || args || source_digest))
//   task digest = hex(BLAKE3("cxx2" || compiler_digest || args || source_digest))
//
// (GetCxxCacheEntryKey, yadcc/daemon/cache_format.cc:56-64; GetCxxTaskDigest, yadcc/daemon/task_digest.cc:25-30.)
// BLAKE3 is written from its published specification (O'Connor, Aumasson, Neves, Wilcox-O'Hearn, "BLAKE3", 2020):
// unkeyed hashing, 32 bytes of output.  One thread hashes one message: it streams the message's 64-byte blocks straight
// from the four pieces (the prefix, the compiler digest in the env table, the argument string in the call's arena, the
// source digest record), so no message is ever assembled, and writes the hex where the filter stages read their keys
// (k_bloom at stride 81, k_rt_find at stride 64).  Messages longer than one 1024-byte chunk are hashed as BLAKE3's tree:
// each completed chunk's chaining value is pushed on a stack and merged into parents once per trailing zero bit of the
// chunk count; the last chunk is folded into what is left on the stack, the root flag on the final compression.
#pragma once
#include "common.cuh"
#include "ydkeys.h"

namespace yd {

// A message is at most the 16-byte prefix + two digests of YD_KEYS_MAX_DIGEST_LEN + one argument string of
// YD_KEYS_MAX_ARGS_LEN; the stack holds one chaining value per set bit of the completed-chunk count.
constexpr uint32_t kB3MaxMsg = 16 + 2 * YD_KEYS_MAX_DIGEST_LEN + YD_KEYS_MAX_ARGS_LEN;
constexpr int kB3Stack = 9;
static_assert((kB3MaxMsg + 1023) / 1024 <= (1u << kB3Stack), "BLAKE3 chaining-value stack too small for the limits");

__device__ __constant__ uint32_t kB3Iv[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                                             0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
__device__ __align__(16) const char kB3CachePrefix[16] = {'u', 's', 'i', 'n', 'g', '-', 'e', 'x',
                                                           't', 'r', 'a', '-', 'i', 'n', 'f', 'o'};
__device__ __align__(16) const char kB3DigestPrefix[4] = {'c', 'x', 'x', '2'};
__device__ __align__(16) const char kB3KeyHead[17] = {'y', 'a', 'd', 'c', 'c', '-', 'c', 'x', 'x',
                                                       '2', '-', 'e', 'n', 't', 'r', 'y', '-'};
enum : uint32_t { kB3ChunkStart = 1, kB3ChunkEnd = 2, kB3Parent = 4, kB3Root = 8 };

struct KeySources {
  const unsigned char* env_bytes;  // the env table: digest e = env_bytes[env_off[e] .. env_off[e + 1])
  const uint32_t* env_off;
  const unsigned char* args;       // the call's argument strings, back to back
  const unsigned long long* args_off;
  const uint32_t* args_index;      // per request
  const unsigned char* src;        // per request: src + i * src_stride, src_len bytes
  unsigned long long src_stride;
  uint32_t src_len;
  const yd_task_req* reqs;         // per request: env_id
  uint32_t n;
  uint32_t both;                   // 1: thread 2i derives request i's cache key, 2i + 1 its task digest
  unsigned char* cache_keys;       // n x YD_KEYS_CACHE_KEY_LEN, or null
  unsigned char* task_digests;     // n x YD_KEYS_TASK_DIGEST_LEN, or null
};

__device__ __forceinline__ void B3G(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, uint32_t x, uint32_t y) {
  a += b + x; d = __funnelshift_r(d ^ a, d ^ a, 16);
  c += d;     b = __funnelshift_r(b ^ c, b ^ c, 12);
  a += b + y; d = __funnelshift_r(d ^ a, d ^ a, 8);
  c += d;     b = __funnelshift_r(b ^ c, b ^ c, 7);
}

// The compression function's first eight output words: cv <- compress(cv, m, counter, len, flags).  m is permuted in
// place between the rounds (its contents are not needed afterwards).
__device__ __forceinline__ void B3Compress(uint32_t cv[8], uint32_t m[16], uint32_t counter, uint32_t len, uint32_t flags) {
  uint32_t v[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7],
                    kB3Iv[0], kB3Iv[1], kB3Iv[2], kB3Iv[3], counter, 0u, len, flags};  // (counter < 2^32 here)
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    B3G(v[0], v[4], v[8], v[12], m[0], m[1]);
    B3G(v[1], v[5], v[9], v[13], m[2], m[3]);
    B3G(v[2], v[6], v[10], v[14], m[4], m[5]);
    B3G(v[3], v[7], v[11], v[15], m[6], m[7]);
    B3G(v[0], v[5], v[10], v[15], m[8], m[9]);
    B3G(v[1], v[6], v[11], v[12], m[10], m[11]);
    B3G(v[2], v[7], v[8], v[13], m[12], m[13]);
    B3G(v[3], v[4], v[9], v[14], m[14], m[15]);
    if (r < 6) {  // message permutation 2 6 3 10 7 0 4 13 1 11 12 5 9 14 15 8 (register renaming only)
      const uint32_t t0 = m[0], t1 = m[1], t2 = m[2], t3 = m[3], t4 = m[4], t5 = m[5], t6 = m[6], t7 = m[7],
                     t8 = m[8], t9 = m[9], t10 = m[10], t11 = m[11], t12 = m[12], t13 = m[13], t14 = m[14], t15 = m[15];
      m[0] = t2; m[1] = t6; m[2] = t3; m[3] = t10; m[4] = t7; m[5] = t0; m[6] = t4; m[7] = t13;
      m[8] = t1; m[9] = t11; m[10] = t12; m[11] = t5; m[12] = t9; m[13] = t14; m[14] = t15; m[15] = t8;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) cv[i] = v[i] ^ v[i + 8];
}

// Little-endian word at an arbitrary byte address: two aligned loads and a funnel shift.  Both loads stay inside the
// aligned words that hold p[0..3], so nothing past the piece's last word is read.
__device__ __forceinline__ uint32_t LoadU32(const unsigned char* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = uint32_t(a & 3) * 8;
  const uint32_t lo = __ldg(w);
  return sh ? __funnelshift_r(lo, __ldg(w + 1), sh) : lo;
}

struct B3Msg {
  const unsigned char* ptr[4];  // prefix, compiler digest, argument string, source digest
  uint32_t end[4];              // running ends: piece k = [end[k-1], end[k])
};

// Message word at byte position p (bytes past the message read as zero, as BLAKE3 pads its last block).
__device__ __forceinline__ uint32_t MsgWord(const B3Msg& g, uint32_t p) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t s = k ? g.end[k - 1] : 0u;
    if (p >= s && p + 4 <= g.end[k]) return LoadU32(g.ptr[k] + (p - s));
  }
  uint32_t w = 0;  // the word straddles a piece boundary or the message's end
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const uint32_t q = p + b;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t s = k ? g.end[k - 1] : 0u;
      if (q >= s && q < g.end[k]) w |= uint32_t(__ldg(g.ptr[k] + (q - s))) << (8 * b);
    }
  }
  return w;
}

// BLAKE3 of the message, as eight little-endian words.
__device__ __forceinline__ void B3Hash(const B3Msg& g, uint32_t out[8]) {
  uint32_t stack[kB3Stack][8];
  int depth = 0;
  const uint32_t L = g.end[3];
  const uint32_t n_chunks = L ? (L + 1023) / 1024 : 1;
  for (uint32_t c = 0; c < n_chunks; ++c) {
    uint32_t cv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) cv[i] = kB3Iv[i];
    const uint32_t clen = min(1024u, L - c * 1024);
    const uint32_t n_blocks = clen ? (clen + 63) / 64 : 1;
    const bool last_chunk = c + 1 == n_chunks;
    for (uint32_t b = 0; b < n_blocks; ++b) {
      uint32_t m[16];
      const uint32_t p = c * 1024 + b * 64;
#pragma unroll
      for (int i = 0; i < 16; ++i) m[i] = MsgWord(g, p + 4 * i);
      uint32_t flags = (b == 0 ? kB3ChunkStart : 0u) | (b + 1 == n_blocks ? kB3ChunkEnd : 0u);
      if (last_chunk && b + 1 == n_blocks && depth == 0) flags |= kB3Root;  // a one-chunk message: this is the root
      B3Compress(cv, m, c, min(64u, clen - b * 64), flags);
    }
    // completed chunks are pushed, merging one parent per trailing zero of the count; the last chunk folds the stack
    uint32_t total = c + 1;
    while (depth > 0 && (last_chunk || (total & 1) == 0)) {
      --depth;
      uint32_t m[16];
#pragma unroll
      for (int i = 0; i < 8; ++i) { m[i] = stack[depth][i]; m[i + 8] = cv[i]; }
#pragma unroll
      for (int i = 0; i < 8; ++i) cv[i] = kB3Iv[i];
      B3Compress(cv, m, 0, 64, kB3Parent | (last_chunk && depth == 0 ? kB3Root : 0u));
      total >>= 1;
    }
    if (!last_chunk) {
#pragma unroll
      for (int i = 0; i < 8; ++i) stack[depth][i] = cv[i];
      ++depth;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) out[i] = cv[i];
    }
  }
}

__global__ void __launch_bounds__(128) k_task_keys(KeySources k) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = k.both ? t >> 1 : t;
  if (i >= k.n) return;
  const bool cache = k.both ? (t & 1) == 0 : k.cache_keys != nullptr;
  const uint32_t env = k.reqs[i].env_id;
  const uint32_t a = k.args_index[i];
  const unsigned long long a0 = k.args_off[a];
  const uint32_t e0 = k.env_off[env], e1 = k.env_off[env + 1];
  B3Msg g;
  g.ptr[0] = reinterpret_cast<const unsigned char*>(cache ? kB3CachePrefix : kB3DigestPrefix);
  g.ptr[1] = k.env_bytes + e0;
  g.ptr[2] = k.args + a0;
  g.ptr[3] = k.src + i * k.src_stride;
  g.end[0] = cache ? 16u : 4u;
  g.end[1] = g.end[0] + (e1 - e0);
  g.end[2] = g.end[1] + uint32_t(k.args_off[a + 1] - a0);
  g.end[3] = g.end[2] + k.src_len;
  uint32_t h[8];
  B3Hash(g, h);
  unsigned char* o = cache ? k.cache_keys + size_t(i) * YD_KEYS_CACHE_KEY_LEN : k.task_digests + size_t(i) * YD_KEYS_TASK_DIGEST_LEN;
  if (cache) {
#pragma unroll
    for (int j = 0; j < 17; ++j) o[j] = kB3KeyHead[j];
    o += 17;
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const uint32_t byte = (h[j >> 2] >> (8 * (j & 3))) & 0xffu;
    const uint32_t hi = byte >> 4, lo = byte & 15;
    o[2 * j] = (unsigned char)(hi < 10 ? '0' + hi : 'a' - 10 + hi);
    o[2 * j + 1] = (unsigned char)(lo < 10 ? '0' + lo : 'a' - 10 + lo);
  }
}

}  // namespace yd
