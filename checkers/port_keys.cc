// port_keys.cc -- TEST INFRASTRUCTURE: the CPU restatement (oracle/port.cc) plus the task keys of a delegate
// (yd_derive_task_keys, yd_derive_filter_and_wait_for_starting_new_tasks), exported as checkers/libydport_keys.so.
// BLAKE3 is restated here from its published specification, as port.cc restates XXH64; it is pinned against the
// reference's own BLAKE3 (oracle/ref_keys.cc) by tests/test_task_keys.py.
#include <array>
#include <initializer_list>
#include <string_view>

#include "../oracle/port.cc"
#include "ydsched_keys_impl.inc"

// ---- task keys (yd_derive_task_keys): BLAKE3 restated from its published specification ---------------------------
// (J. O'Connor, J.-P. Aumasson, S. Neves, Z. Wilcox-O'Hearn, "BLAKE3", 2020, sections 2.1-2.6): an incremental hasher
// with the chaining-value stack merged by the chunk counter; unkeyed, 32 bytes of output.
namespace {

constexpr uint32_t kB3Iv[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                               0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
constexpr int kB3Perm[16] = {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8};
enum : uint32_t { kChunkStart = 1, kChunkEnd = 2, kParent = 4, kRoot = 8 };

inline uint32_t Rotr(uint32_t x, int r) { return (x >> r) | (x << (32 - r)); }

void B3G(uint32_t* v, int a, int b, int c, int d, uint32_t x, uint32_t y) {
  v[a] += v[b] + x; v[d] = Rotr(v[d] ^ v[a], 16);
  v[c] += v[d];     v[b] = Rotr(v[b] ^ v[c], 12);
  v[a] += v[b] + y; v[d] = Rotr(v[d] ^ v[a], 8);
  v[c] += v[d];     v[b] = Rotr(v[b] ^ v[c], 7);
}

// compression function, first 8 output words (the chaining value)
void B3Compress(const uint32_t cv[8], const uint32_t block[16], uint64_t counter, uint32_t len, uint32_t flags,
                uint32_t out[8]) {
  uint32_t v[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], kB3Iv[0], kB3Iv[1], kB3Iv[2], kB3Iv[3],
                    (uint32_t)counter, (uint32_t)(counter >> 32), len, flags};
  uint32_t m[16];
  memcpy(m, block, sizeof m);
  for (int r = 0; r != 7; ++r) {
    B3G(v, 0, 4, 8, 12, m[0], m[1]);   B3G(v, 1, 5, 9, 13, m[2], m[3]);
    B3G(v, 2, 6, 10, 14, m[4], m[5]);  B3G(v, 3, 7, 11, 15, m[6], m[7]);
    B3G(v, 0, 5, 10, 15, m[8], m[9]);  B3G(v, 1, 6, 11, 12, m[10], m[11]);
    B3G(v, 2, 7, 8, 13, m[12], m[13]); B3G(v, 3, 4, 9, 14, m[14], m[15]);
    uint32_t p[16];
    for (int i = 0; i != 16; ++i) p[i] = m[kB3Perm[i]];
    memcpy(m, p, sizeof m);
  }
  for (int i = 0; i != 8; ++i) out[i] = v[i] ^ v[i + 8];
}

class Blake3Hasher {
 public:
  void Update(const char* p, size_t len) {
    while (len) {
      if (buf_len_ == 64) {  // a full block is compressed only once more input shows it is not the chunk's last
        Flush();
      }
      const size_t take = std::min(len, size_t(64) - buf_len_);
      memcpy(buf_ + buf_len_, p, take);
      buf_len_ += take; p += take; len -= take;
    }
  }
  void Hex(char* dst) {  // finalizes; writes 64 lowercase hex digits
    // the current chunk's last block is the output node unless chunks were completed before it
    uint32_t block[16];
    Words(block);
    uint32_t flags = kChunkEnd | (blocks_ == 0 ? kChunkStart : 0);
    uint32_t out[8];
    if (stack_.empty()) {
      B3Compress(cv_, block, chunk_, (uint32_t)buf_len_, flags | kRoot, out);
    } else {
      B3Compress(cv_, block, chunk_, (uint32_t)buf_len_, flags, out);
      for (size_t k = stack_.size(); k-- != 0;) {
        uint32_t pb[16];
        memcpy(pb, stack_[k].data(), 32);
        memcpy(pb + 8, out, 32);
        B3Compress(kB3Iv, pb, 0, 64, kParent | (k == 0 ? kRoot : 0), out);
      }
    }
    static const char kHex[] = "0123456789abcdef";
    for (int i = 0; i != 32; ++i) {
      const uint8_t b = uint8_t(out[i / 4] >> (8 * (i % 4)));
      dst[2 * i] = kHex[b >> 4];
      dst[2 * i + 1] = kHex[b & 15];
    }
  }

 private:
  void Words(uint32_t* w) const {
    uint8_t b[64] = {};
    memcpy(b, buf_, buf_len_);
    for (int i = 0; i != 16; ++i) w[i] = b[4 * i] | b[4 * i + 1] << 8 | b[4 * i + 2] << 16 | uint32_t(b[4 * i + 3]) << 24;
  }
  void Flush() {
    uint32_t block[16];
    Words(block);
    const uint32_t flags = (blocks_ == 0 ? kChunkStart : 0) | (blocks_ == 15 ? kChunkEnd : 0);
    B3Compress(cv_, block, chunk_, 64, flags, cv_);
    buf_len_ = 0;
    if (++blocks_ == 16) {  // chunk complete: push its chaining value, merging one parent per trailing zero of the count
      std::array<uint32_t, 8> cv;
      memcpy(cv.data(), cv_, 32);
      uint64_t total = ++chunk_;
      while ((total & 1) == 0) {
        uint32_t pb[16];
        memcpy(pb, stack_.back().data(), 32);
        memcpy(pb + 8, cv.data(), 32);
        B3Compress(kB3Iv, pb, 0, 64, kParent, cv.data());
        stack_.pop_back();
        total >>= 1;
      }
      stack_.push_back(cv);
      memcpy(cv_, kB3Iv, 32);
      blocks_ = 0;
    }
  }
  uint32_t cv_[8] = {kB3Iv[0], kB3Iv[1], kB3Iv[2], kB3Iv[3], kB3Iv[4], kB3Iv[5], kB3Iv[6], kB3Iv[7]};
  uint8_t buf_[64];
  size_t buf_len_ = 0;
  uint32_t blocks_ = 0;  // blocks of the current chunk already compressed
  uint64_t chunk_ = 0;   // index of the current chunk
  std::vector<std::array<uint32_t, 8>> stack_;
};

void B3Hex(std::initializer_list<std::string_view> pieces, char* dst) {
  Blake3Hasher h;
  for (auto&& p : pieces) h.Update(p.data(), p.size());
  h.Hex(dst);
}

}  // namespace

extern "C" int yd_derive_task_keys(yd_sched* s, const yd_task_req* reqs, size_t n, const yd_task_sources* src,
                                   char* cache_keys_out, char* task_digests_out) {
  if (int rc = yd_keys_check(s->envs, reqs, n, src)) return rc;
  for (size_t i = 0; i != n; ++i) {
    const std::string_view env = s->envs[reqs[i].env_id];
    const uint32_t a = src->args_index[i];
    const std::string_view args(src->args + src->args_offsets[a], src->args_offsets[a + 1] - src->args_offsets[a]);
    const std::string_view sd(src->source_digests + i * src->source_digest_stride, src->source_digest_len);
    if (cache_keys_out) {
      char* k = cache_keys_out + i * YD_KEYS_CACHE_KEY_LEN;
      memcpy(k, "yadcc-cxx2-entry-", 17);
      B3Hex({"using-extra-info", env, args, sd}, k + 17);
    }
    if (task_digests_out) B3Hex({"cxx2", env, args, sd}, task_digests_out + i * YD_KEYS_TASK_DIGEST_LEN);
  }
  return YD_KEYS_OK;
}

#include "ydsched_derive_impl.inc"
