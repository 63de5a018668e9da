// Host wrappers around the product's device primitives, for tests/test_device_primitives.py (loaded with ctypes).
//
// Each wrapper takes host arrays, allocates the device buffers and the zeroed scratch the way the product's launch
// sites do, launches the product's own kernels (the headers below, through the same host sequences as the product:
// yd::rs_sort, yd::keep_count_scan, yd::keep_scatter), copies the results back and returns the cudaError_t of the
// launches, checked after a cudaDeviceSynchronize.  Output buffers start filled with 0xFF bytes, so a test also sees
// every word a kernel must not have written.  Built by `make primitives` into tests/kernels/libydprim.so.
#include <cuda_runtime.h>

#include <algorithm>

#include "filter.cuh"
#include "radix.cuh"
#include "state.cuh"

namespace {

#define CK(x)                             \
  do {                                    \
    const cudaError_t e_ = (x);           \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

// A device allocation freed on every return path.
struct Dev {
  void* p = nullptr;
  ~Dev() {
    if (p) cudaFree(p);
  }
  cudaError_t alloc(size_t bytes, int fill) {
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(bytes, 16));
    return e != cudaSuccess ? e : cudaMemset(p, fill, std::max<size_t>(bytes, 16));
  }
  template <class T>
  T* as() const { return static_cast<T*>(p); }
};

// The launches' own error, then the first fault of their execution.
cudaError_t Finish() {
  const cudaError_t e = cudaGetLastError();
  const cudaError_t s = cudaDeviceSynchronize();
  return e != cudaSuccess ? e : s;
}

// n keys (n read on the device), nb tiles, bits [first_bit, last_bit] as LaunchSort takes them.  keys_out / vals_out:
// nb * kRsTile elements each, buffer 0 of the ping-pong after the sort.
template <typename KeyT>
int Sort(const KeyT* keys, unsigned long long n, uint32_t nb, int first_bit, int last_bit, KeyT* keys_out,
         uint32_t* vals_out) {
  const int passes = (last_bit - first_bit) / yd::kRsBits + 1;
  if (passes < 1 || passes > yd::kRsMaxPasses || nb == 0 || n > (unsigned long long)nb * yd::kRsTile) {
    return (int)cudaErrorInvalidValue;
  }
  const size_t cap = size_t(nb) * yd::kRsTile;
  Dev d_in, d_n, d_zero, d_k[2], d_v[2];
  CK(d_in.alloc(n * sizeof(KeyT), 0xFF));
  CK(d_n.alloc(8, 0));
  CK(d_zero.alloc(passes * yd::rs_pass_words(nb) * 4, 0));
  for (int b = 0; b < 2; ++b) {
    CK(d_k[b].alloc(cap * sizeof(KeyT), 0xFF));
    CK(d_v[b].alloc(cap * 4, 0xFF));
  }
  if (n) CK(cudaMemcpy(d_in.p, keys, n * sizeof(KeyT), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_n.p, &n, 8, cudaMemcpyHostToDevice));
  KeyT* const k[2] = {d_k[0].as<KeyT>(), d_k[1].as<KeyT>()};
  uint32_t* const v[2] = {d_v[0].as<uint32_t>(), d_v[1].as<uint32_t>()};
  yd::rs_sort<KeyT>(d_in.as<KeyT>(), d_n.as<unsigned long long>(), nb, first_bit, last_bit, d_zero.as<uint32_t>(), k, v, 0);
  CK(Finish());
  CK(cudaMemcpy(keys_out, k[0], cap * sizeof(KeyT), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(vals_out, v[0], cap * 4, cudaMemcpyDeviceToHost));
  return 0;
}

template <class Req>
int Compact(const Req* reqs, uint32_t n, const uint8_t* bloom_hit, const uint32_t* rt_hit, uint8_t* verdict,
            uint32_t* tile_off, yd_task_req* out) {
  if (n == 0) return (int)cudaErrorInvalidValue;  // the product answers an empty queue without launching
  const uint32_t nt = (n + 1023) / 1024;
  size_t out_cap = 1024;  // the solver's queue: NextPow2(n, 1024) requests
  while (out_cap < n) out_cap *= 2;
  Dev d_in, d_bloom, d_rt, d_verdict, d_tile, d_out;
  CK(d_in.alloc(size_t(n) * sizeof(Req), 0));
  CK(d_verdict.alloc(n, 0xFF));
  CK(d_tile.alloc((nt + 1) * 4, 0xFF));
  CK(d_out.alloc(out_cap * sizeof(yd_task_req), 0xFF));
  CK(cudaMemcpy(d_in.p, reqs, size_t(n) * sizeof(Req), cudaMemcpyHostToDevice));
  if (bloom_hit) {
    CK(d_bloom.alloc(n, 0));
    CK(cudaMemcpy(d_bloom.p, bloom_hit, n, cudaMemcpyHostToDevice));
  }
  if (rt_hit) {
    CK(d_rt.alloc(size_t(n) * 16, 0));
    CK(cudaMemcpy(d_rt.p, rt_hit, size_t(n) * 16, cudaMemcpyHostToDevice));
  }
  yd::keep_count_scan(d_bloom.as<uint8_t>(), d_rt.as<uint4>(), n, d_verdict.as<uint8_t>(), d_tile.as<uint32_t>(), 0);
  yd::keep_scatter(d_in.as<Req>(), d_verdict.as<uint8_t>(), d_tile.as<uint32_t>(), n, d_out.as<yd_task_req>(), 0);
  CK(Finish());
  CK(cudaMemcpy(verdict, d_verdict.p, n, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(tile_off, d_tile.p, (nt + 1) * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out, d_out.p, size_t(n) * sizeof(yd_task_req), cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace

extern "C" {

int yd_prim_sort_u32(const uint32_t* keys, unsigned long long n, uint32_t nb, int first_bit, int last_bit,
                     uint32_t* keys_out, uint32_t* vals_out) {
  return Sort<uint32_t>(keys, n, nb, first_bit, last_bit, keys_out, vals_out);
}

int yd_prim_sort_u64(const unsigned long long* keys, unsigned long long n, uint32_t nb, int first_bit, int last_bit,
                     unsigned long long* keys_out, uint32_t* vals_out) {
  return Sort<unsigned long long>(keys, n, nb, first_bit, last_bit, keys_out, vals_out);
}

// k_scan_u32 over data[0, len) in place, one block as the product launches it: the static length n_static, or with
// use_dyn the device-side length min(n_dyn, dyn_cap) * per_dyn + 1.  *total: the kernel's total (0xFFFFFFFF before).
int yd_prim_scan_u32(uint32_t* data, unsigned long long len, uint32_t n_static, int use_dyn, uint32_t n_dyn,
                     uint32_t per_dyn, uint32_t dyn_cap, uint32_t* total) {
  Dev d_data, d_n, d_total;
  CK(d_data.alloc(len * 4, 0));
  CK(d_n.alloc(4, 0));
  CK(d_total.alloc(4, 0xFF));
  if (len) CK(cudaMemcpy(d_data.p, data, len * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_n.p, &n_dyn, 4, cudaMemcpyHostToDevice));
  yd::k_scan_u32<<<1, 1024>>>(d_data.as<uint32_t>(), n_static, use_dyn ? d_n.as<uint32_t>() : nullptr, per_dyn,
                              d_total.as<uint32_t>(), dyn_cap);
  CK(Finish());
  if (len) CK(cudaMemcpy(data, d_data.p, len * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(total, d_total.p, 4, cudaMemcpyDeviceToHost));
  return 0;
}

// k_scan_rows over data[0, len) in place: `grid` blocks (at most 256, the co-resident bound the kernel relies on),
// min(n_rows, grid) rows of per_row counts, and its mailboxes: grid + 1 zeroed 64-bit words.
int yd_prim_scan_rows(uint32_t* data, unsigned long long len, uint32_t grid, uint32_t n_rows, uint32_t per_row) {
  if (grid == 0 || grid > 256) return (int)cudaErrorInvalidValue;
  Dev d_data, d_n, d_pub;
  CK(d_data.alloc(len * 4, 0));
  CK(d_n.alloc(4, 0));
  CK(d_pub.alloc((grid + 1) * 8, 0));
  if (len) CK(cudaMemcpy(d_data.p, data, len * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_n.p, &n_rows, 4, cudaMemcpyHostToDevice));
  yd::k_scan_rows<<<grid, 1024>>>(d_data.as<uint32_t>(), d_n.as<uint32_t>(), per_row, d_pub.as<unsigned long long>());
  CK(Finish());
  if (len) CK(cudaMemcpy(data, d_data.p, len * 4, cudaMemcpyDeviceToHost));
  return 0;
}

// The pre-filtered queue's compaction of n >= 1 requests (24-byte records, or 16-byte ones with req16).  bloom_hit (n
// bytes) and rt_hit (n yd_running_hit records as four words each) may be null.  Out: the verdicts, the ceil(n / 1024) + 1
// scanned tile counts, and the first n records of the solver's queue.
int yd_prim_compact(int req16, const void* reqs, uint32_t n, const uint8_t* bloom_hit, const uint32_t* rt_hit,
                    uint8_t* verdict, uint32_t* tile_off, yd_task_req* out) {
  return req16 ? Compact(static_cast<const yd_task_req16*>(reqs), n, bloom_hit, rt_hit, verdict, tile_off, out)
               : Compact(static_cast<const yd_task_req*>(reqs), n, bloom_hit, rt_hit, verdict, tile_off, out);
}

// k_state_merge of W lists of 24-byte lease records at lists + q * stride (counts[q] each), launched as the group
// export does.  out: out_len records, of which the first sum(counts) are the merged list.
int yd_prim_state_merge(const yd::StateLease* lists, unsigned long long stride, const unsigned long long* counts,
                        uint32_t W, yd::StateLease* out, unsigned long long out_len) {
  if (stride == 0 || W == 0) return (int)cudaErrorInvalidValue;
  Dev d_lists, d_counts, d_out;
  CK(d_lists.alloc(stride * W * sizeof(yd::StateLease), 0));
  CK(d_counts.alloc(W * 8, 0));
  CK(d_out.alloc(out_len * sizeof(yd::StateLease), 0xFF));
  CK(cudaMemcpy(d_lists.p, lists, stride * W * sizeof(yd::StateLease), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_counts.p, counts, W * 8, cudaMemcpyHostToDevice));
  const unsigned long long threads = stride * W;
  yd::k_state_merge<<<(unsigned)((threads + 255) / 256), 256>>>(d_lists.as<yd::StateLease>(), stride,
                                                                 d_counts.as<unsigned long long>(), W,
                                                                 d_out.as<yd::StateLease>());
  CK(Finish());
  if (out_len) CK(cudaMemcpy(out, d_out.p, out_len * sizeof(yd::StateLease), cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
