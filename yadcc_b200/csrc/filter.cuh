// filter.cuh -- the delegate-side pre-filters of BASELINE configs[3] fused in front of the solve.
//
// Before a delegate daemon asks the scheduler for a grant it (1) consults the compilation cache's bloom filter
// (yadcc/daemon/local/distributed_cache_reader.cc:70-77: a possible hit is served from the cache, no grant is asked) and
// (2) looks the task's digest up among the tasks already running (running_task_keeper.cc:67-75, caller
// distributed_task_dispatcher.cc:257: an identical translation unit being compiled somewhere is joined).  Only what
// passes both is offered to the scheduler.  With the whole queue in HBM the three stages are one pipeline: bloom
// probes (bloom.cuh), index probes (running_index.cuh), an order-preserving compaction of the survivors (here), the
// solve.
//
//   k_keep_count    verdict per request (0 offered, 1 cache hit, 2 joined) + survivors per tile of 1024
//   (k_scan_u32     exclusive scan of the tile counts, total behind them)
//   k_keep_scatter  survivors -> the solver's queue, FIFO order kept (16-byte requests are unpacked on the way)
#pragma once
#include "common.cuh"
#include "radix.cuh"  // k_scan_u32

namespace yd {

__global__ void __launch_bounds__(1024) k_keep_count(const uint8_t* __restrict__ bloom_hit /* may be null */,
                                                     const uint4* __restrict__ rt_hit /* yd_running_hit, may be null */,
                                                     uint32_t n, uint8_t* __restrict__ verdict,
                                                     uint32_t* __restrict__ tile_cnt) {
  __shared__ uint32_t warp_cnt[32];
  const uint32_t q = blockIdx.x * 1024 + threadIdx.x;
  uint32_t v = 3;  // beyond the queue's end
  if (q < n) {
    v = (bloom_hit && bloom_hit[q]) ? 1u : (rt_hit && rt_hit[q].w) ? 2u : 0u;  // the cache is consulted first
    verdict[q] = (uint8_t)v;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, v == 0);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = __popc(bal);
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t c = __reduce_add_sync(0xffffffffu, warp_cnt[threadIdx.x]);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = c;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) tile_cnt[gridDim.x] = 0;  // the scan's end cell
}

// A survivor into the solver's queue: a 24-byte request as it is, a 16-byte one (yd_task_req16) unpacked.
__device__ __forceinline__ void keep_put(const yd_task_req* __restrict__ in, yd_task_req* __restrict__ out) {
  const uint2* src = reinterpret_cast<const uint2*>(in);
  uint2* dst = reinterpret_cast<uint2*>(out);
  dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
}
__device__ __forceinline__ void keep_put(const yd_task_req16* __restrict__ in, yd_task_req* __restrict__ out) {
  const uint4 w = *reinterpret_cast<const uint4*>(in);
  uint2* dst = reinterpret_cast<uint2*>(out);
  const unsigned long long ns = (unsigned long long)(w.w & 0x7fffffffu) * 1000000ull;
  dst[0] = make_uint2(w.x, w.y);
  dst[1] = make_uint2(w.z, (w.w & YD_LEASE_PREFETCH) ? YD_REQ_FLAG_PREFETCH : 0u);
  dst[2] = make_uint2((uint32_t)ns, (uint32_t)(ns >> 32));
}

template <class Req>
__global__ void __launch_bounds__(1024) k_keep_scatter(const Req* __restrict__ in, const uint8_t* __restrict__ verdict,
                                                       const uint32_t* __restrict__ tile_off, uint32_t n,
                                                       yd_task_req* __restrict__ out) {
  __shared__ uint32_t warp_cnt[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t q = blockIdx.x * 1024 + tid;
  const bool keep = q < n && verdict[q] == 0;
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  if (!keep) return;
  uint32_t before = tile_off[blockIdx.x];
  for (uint32_t w = 0; w < warp; ++w) before += warp_cnt[w];
  before += __popc(bal & ((1u << lane) - 1));
  keep_put(in + q, out + before);
}

// The compaction's first two launches on `st`, for a queue of n >= 1 requests (callers answer an empty queue without
// launching): the verdicts, and in tile_off (ceil(n / 1024) + 1 words) the survivors' offsets per tile of 1024 with
// their total behind them.
inline void keep_count_scan(const uint8_t* bloom_hit, const uint4* rt_hit, uint32_t n, uint8_t* verdict, uint32_t* tile_off,
                            cudaStream_t st) {
  const uint32_t nt = (n + 1023) / 1024;
  k_keep_count<<<nt, 1024, 0, st>>>(bloom_hit, rt_hit, n, verdict, tile_off);
  k_scan_u32<<<1, 1024, 0, st>>>(tile_off, nt + 1, nullptr, 0, nullptr, 0);
}

// Its last launch: the survivors of `in` (n requests, verdicts and tile offsets from keep_count_scan) -> out, in order.
template <class Req>
inline void keep_scatter(const Req* in, const uint8_t* verdict, const uint32_t* tile_off, uint32_t n, yd_task_req* out,
                         cudaStream_t st) {
  k_keep_scatter<<<(n + 1023) / 1024, 1024, 0, st>>>(in, verdict, tile_off, n, out);
}

}  // namespace yd
