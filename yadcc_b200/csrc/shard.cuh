// shard.cuh -- device helpers of the range-sharded scheduler (include/ydshard.h).
//
// The solve itself is the ordinary slot-stream pipeline (slots.cuh, radix.cuh, classes.cuh,
// parallel.cuh, solve_merge.cuh); these kernels sit at its four exchange points.
#pragma once
#include "classes.cuh"
#include "solve_merge.cuh"

namespace yd {

// Exchange 4 payload, one u32 array all-reduced with SUM:
//   [0, S)            slots claimed on each servant by THIS rank's requests
//   [S, S + world)    cell `rank` = grants of this rank (the sum is an all-gather)
//   [S + world + 0]   batches that must be handed back (any rank says so -> everybody stands down)
//   [S + world + 1]   chunks re-run in the merge solver's last round (identical on all ranks; summed anyway)
constexpr uint32_t kShardTail = 8;

// This rank's verdict on the batch: a component that only the sequential solver can decide (mode 0
// with requests, or handed back by the merge solver), or any earlier overflow flag.
__global__ void __launch_bounds__(256) k_shard_flags(ClassTable ct, const uint32_t* __restrict__ comp_mode,
                                                     const uint32_t* __restrict__ viol, uint32_t n_comps,
                                                     uint32_t* __restrict__ tail) {
  __shared__ uint32_t s_bad;
  if (threadIdx.x == 0) s_bad = ct.meta[1] ? 1u : 0u;
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < n_comps; c += blockDim.x) {
    if ((comp_mode[c] == 0 && ct.comp_ncls[c] != 0) || viol[c]) s_bad = 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) tail[0] = s_bad;
}

// After exchange 4: where this rank's grants start in the batch's FIFO numbering, the batch's total,
// and the common stand-down flag (meta[1] != 0 makes the final kernels leave all state alone).
__global__ void k_shard_post(const uint32_t* __restrict__ sums, uint32_t S, uint32_t rank, uint32_t world,
                             uint32_t* __restrict__ meta, uint32_t* __restrict__ prefix_total) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t before = 0, all = 0;
  for (uint32_t g = 0; g < world; ++g) {
    const uint32_t v = sums[S + g];
    if (g < rank) before += v;
    all += v;
  }
  prefix_total[0] = before;
  prefix_total[1] = all;
  prefix_total[2] = sums[S + world];  // ranks that want the batch handed back
  if (sums[S + world] != 0 && meta[1] == 0) meta[1] = 4;
}

// k_final_count leaves the per-block grant counts; their sum is this rank's grant count.
__global__ void __launch_bounds__(1024) k_shard_count_grants(const uint32_t* __restrict__ block_counts, uint32_t nb,
                                                            const uint32_t* __restrict__ abort_flag,
                                                            uint32_t* __restrict__ cell) {
  __shared__ uint32_t s_sum;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  uint32_t mine = 0;
  if (!(abort_flag && *abort_flag)) {
    for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) mine += block_counts[i];
  }
  if (mine) atomicAdd(&s_sum, mine);
  __syncthreads();
  if (threadIdx.x == 0) *cell = s_sum;
}

// running_tasks decrements made on one rank only -- a lease lives on the rank that holds its request, so a zombie
// swept by a heartbeat (k_notify_sweep) or a freed lease (k_free) lowers running_tasks there first -- reach the other
// ranks at the next collective call: `parts` holds every rank's decrements (`nparts` arrays `stride` words apart, or
// their sum), `dec` this rank's own, already applied to `run`.
__global__ void k_run_reconcile(uint32_t S, const uint32_t* __restrict__ parts, size_t stride, uint32_t nparts,
                                uint32_t* __restrict__ dec, uint32_t* __restrict__ run) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  uint32_t all = 0;
  for (uint32_t g = 0; g < nparts; ++g) all += parts[g * stride + s];
  run[s] -= all - dec[s];
  dec[s] = 0;
}

}  // namespace yd
