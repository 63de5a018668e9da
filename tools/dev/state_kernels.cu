// Device time of the range-sharded state kernels (state.cuh) for tools/time_shard_state.py: k_state_merge over W
// all-gathered record lists of n leases in all (each id on a seeded random rank, the lists padded to the longest, as
// yd_shard_export_state lays them out) and k_state_scatter of n records into a ring, materialising rank 0's block of
// n / W.  CUDA events around each launch; `reps` launches each, after one warm-up launch.  Built by the tool with nvcc
// into a temporary directory; loaded with ctypes.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>

#include "state.cuh"

#define CK(x)                                                                       \
  do {                                                                              \
    cudaError_t e = (x);                                                            \
    if (e != cudaSuccess) {                                                         \
      fprintf(stderr, "%s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      return 1;                                                                     \
    }                                                                               \
  } while (0)

extern "C" int time_state_kernels(unsigned long long n, unsigned W, unsigned servants, int reps, float* merge_ms,
                                  float* scatter_ms) {
  std::mt19937_64 rng(7);
  std::vector<std::vector<yd::StateLease>> lists(W);
  for (unsigned long long id = 0; id != n; ++id)
    lists[rng() % W].push_back(yd::StateLease{id, (uint32_t)(rng() % servants), 0u, 30000000000ll});
  size_t maxn = 1;
  for (auto& l : lists) maxn = std::max(maxn, l.size());
  std::vector<yd::StateLease> host(maxn * W);
  std::vector<unsigned long long> counts(W);
  for (unsigned r = 0; r != W; ++r) {
    std::copy(lists[r].begin(), lists[r].end(), host.begin() + r * maxn);
    counts[r] = lists[r].size();
  }
  yd::StateLease *d_lists, *d_out;
  unsigned long long* d_counts;
  CK(cudaMalloc(&d_lists, host.size() * sizeof(yd::StateLease)));
  CK(cudaMalloc(&d_out, n * sizeof(yd::StateLease)));
  CK(cudaMalloc(&d_counts, W * 8));
  CK(cudaMemcpy(d_lists, host.data(), host.size() * sizeof(yd::StateLease), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_counts, counts.data(), W * 8, cudaMemcpyHostToDevice));
  // the ring of the scatter: the window of n ids, twice its size rounded up to a power of two
  unsigned long long cap = 1ull << 16;
  while (cap < 2 * n) cap <<= 1;
  yd::TaskRing ring{};
  CK(cudaMalloc(&ring.exp, cap * 8));
  CK(cudaMalloc(&ring.srv, cap * 4));
  CK(cudaMalloc(&ring.flags, cap * 4));
  ring.mask = cap - 1;
  ring.lo = 0;
  ring.next = n;
  ring.id_stride = 1;
  ring.id_offset = 0;
  uint32_t* d_run;
  CK(cudaMalloc(&d_run, servants * 4));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  const unsigned merge_blocks = (unsigned)((maxn * W + 255) / 256), scatter_blocks = (unsigned)((n + 255) / 256);
  for (int k = -1; k < reps; ++k) {
    CK(cudaEventRecord(a));
    yd::k_state_merge<<<merge_blocks, 256>>>(d_lists, maxn, d_counts, W, d_out);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    if (k >= 0) CK(cudaEventElapsedTime(&merge_ms[k], a, b));
    CK(cudaMemset(ring.flags, 0, cap * 4));
    CK(cudaMemset(d_run, 0, servants * 4));
    CK(cudaEventRecord(a));
    yd::k_state_scatter<<<scatter_blocks, 256>>>(d_out, (uint32_t)n, 0u, (uint32_t)((n + W - 1) / W), ring, 0ll, d_run);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    if (k >= 0) CK(cudaEventElapsedTime(&scatter_ms[k], a, b));
  }
  CK(cudaGetLastError());
  // the merge put every record at its id (ids are 0 .. n-1)
  std::vector<yd::StateLease> back(n);
  CK(cudaMemcpy(back.data(), d_out, n * sizeof(yd::StateLease), cudaMemcpyDeviceToHost));
  int bad = 0;
  for (unsigned long long i = 0; i != n; ++i) bad |= back[i].id != i;
  cudaFree(d_lists); cudaFree(d_out); cudaFree(d_counts); cudaFree(ring.exp); cudaFree(ring.srv); cudaFree(ring.flags);
  cudaFree(d_run);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  return bad ? 2 : 0;
}
