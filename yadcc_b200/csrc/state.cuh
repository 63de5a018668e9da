// state.cuh -- the lease part of yd_export_state / yd_import_state (include/ydstate.h).
//
// The lease count is what scales (a million and more at configs[2] / [4] scale), so both directions
// run on the device:
//   export  one pass over the ring's live window [lo, next): per 1024-id block a ballot count of the
//           live leases (k_state_count), the exclusive scan of the block counts (k_final_scan of
//           tasks.cuh, into a scratch Counters), and the compacted 24-byte records in id order
//           (k_state_write), which leave the device in one copy;
//   import  one thread per record: scatter into t_exp / t_srv / t_flags and count the lease into its
//           servant's running_tasks (the per-servant histogram that run[] is).
#pragma once
#include "common.cuh"
#include "ydstate.h"

namespace yd {

struct StateLease {  // ydstate::Lease, the format's 24-byte record
  unsigned long long id;
  uint32_t servant, flags;
  long long expires_rel;
};
static_assert(sizeof(StateLease) == 24, "lease records are 24 bytes");

__device__ __forceinline__ bool state_live(const TaskRing& ring, unsigned long long id) {
  return id < ring.next && (ring.flags[id & ring.mask] & kTaskAlive);
}

// Live leases per block of 1024 ids of the window.
__global__ void __launch_bounds__(1024) k_state_count(TaskRing ring, uint32_t* __restrict__ block_counts) {
  const unsigned long long id = ring.lo + (unsigned long long)blockIdx.x * 1024 + threadIdx.x;
  __shared__ uint32_t warp_cnt[32];
  const uint32_t bal = __ballot_sync(0xffffffffu, state_live(ring, id));
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = __popc(bal);
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t c = __reduce_add_sync(0xffffffffu, warp_cnt[threadIdx.x]);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
  }
}

// The live leases of the window as records, in id order: block b's first record goes to block_off[b].
__global__ void __launch_bounds__(1024) k_state_write(TaskRing ring, long long now_ns, const uint32_t* __restrict__ block_off,
                                                      StateLease* __restrict__ out) {
  const unsigned long long id = ring.lo + (unsigned long long)blockIdx.x * 1024 + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ uint32_t warp_cnt[32];
  const bool live = state_live(ring, id);
  const uint32_t bal = __ballot_sync(0xffffffffu, live);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  if (!live) return;
  uint32_t before = __popc(bal & ((1u << lane) - 1));
  for (uint32_t w = 0; w < warp; ++w) before += warp_cnt[w];
  const uint64_t slot = id & ring.mask;
  const uint32_t f = ring.flags[slot];
  StateLease r;
  r.id = ring.ext(id);
  r.servant = ring.srv[slot];
  r.flags = ((f & kTaskPrefetch) ? YD_STATE_LEASE_PREFETCH : 0u) | ((f & kTaskZombie) ? YD_STATE_LEASE_ZOMBIE : 0u);
  r.expires_rel = ring.exp[slot] - now_ns;
  out[block_off[blockIdx.x] + before] = r;
}

// Import: records -> ring slots, and run[servant] += leases on it.  The ring's flags are zero and
// run[] is zero before the launch.  Leases of one servant tend to sit next to each other (grants of a
// batch), so a warp adds each distinct servant once.
__global__ void k_state_scatter(const StateLease* __restrict__ in, uint32_t n, TaskRing ring, long long now_ns,
                                uint32_t* __restrict__ run) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool have = i < n;
  uint32_t servant = kNone;
  if (have) {
    const StateLease r = in[i];
    unsigned long long local = 0;
    ring.loc(r.id, &local);  // (the host checked that every id is one of ours)
    const uint64_t slot = local & ring.mask;
    ring.exp[slot] = now_ns + r.expires_rel;
    ring.srv[slot] = r.servant;
    ring.flags[slot] = kTaskAlive | ((r.flags & YD_STATE_LEASE_PREFETCH) ? kTaskPrefetch : 0u) |
                       ((r.flags & YD_STATE_LEASE_ZOMBIE) ? kTaskZombie : 0u);
    servant = r.servant;
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, servant);
  if (have && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&run[servant], (uint32_t)__popc(peers));
}

}  // namespace yd
