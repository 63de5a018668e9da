// tasks.cuh -- task-id assignment and the device-resident lease registry.
//
// TaskRegistry (task_dispatcher.h:199-220) is an unordered_map<id, TaskDesc> in
// the reference; every sweep (UnsafeSweepZombiesOf cc:453-476, UnsafeSweepOrphans
// cc:478-496, the zombie marking cc:522-535) walks the whole map under the lock.
// Here ids are dense (next_task_id++ per grant, cc:127), so the registry is a
// power-of-two ring of 16-byte entries in HBM indexed by id & mask; the sweeps
// are coalesced streaming passes over the live window [lo, next).
#pragma once
#include "common.cuh"

namespace yd {

// ---- grants: task ids in FIFO order = exclusive scan over "granted" flags -----

// `abort_flag` (may be null): non-zero means the solver gave up on this batch (class
// table overflow) and the host will rerun it; the final kernels then leave all state alone.
__global__ void __launch_bounds__(1024) k_final_count(const uint32_t* __restrict__ res,
                                                      const DynParams* __restrict__ dp,
                                                      uint32_t* __restrict__ block_counts,
                                                      const uint32_t* __restrict__ abort_flag,
                                                      const uint32_t* __restrict__ comp_sv = nullptr,
                                                      uint32_t* __restrict__ claims = nullptr) {
  if (abort_flag && *abort_flag) return;
  uint32_t q = blockIdx.x * 1024 + threadIdx.x;
  const bool granted = (q < dp->n) && (res[q] < kResTimeout);
  // range-sharded queue: slots this rank's requests claimed, per servant (summed over the ranks afterwards)
  if (claims && granted) atomicAdd(&claims[comp_sv[res[q]]], 1u);
  // ballot + per-warp counters, the same way k_final_write ranks the grants
  // (bar.red-based __syncthreads_count under-counted under compute-sanitizer)
  __shared__ uint32_t warp_cnt[32];
  const uint32_t bal = __ballot_sync(0xffffffffu, granted);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = __popc(bal);
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t c = __reduce_add_sync(0xffffffffu, warp_cnt[threadIdx.x]);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
  }
}

// `id_prefix` (may be null): grants of the lower ranks of a range-sharded queue, i.e. where this rank's
// first grant sits in the batch's FIFO numbering.
__global__ void __launch_bounds__(1024) k_final_scan(uint32_t* __restrict__ block_counts, uint32_t nb,
                                                     Counters* __restrict__ counters,
                                                     const uint32_t* __restrict__ abort_flag,
                                                     const uint32_t* __restrict__ id_prefix = nullptr) {
  if (abort_flag && *abort_flag) return;
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nb; base += 1024) {
    uint32_t i = base + tid;
    uint32_t v = i < nb ? block_counts[i] : 0;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = warp_sums[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    uint32_t carry = carry_s;
    if (i < nb) block_counts[i] = (id_prefix ? *id_prefix : 0u) + carry + (warp ? warp_sums[warp - 1] : 0) + x - v;  // exclusive
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_sums[31];
    __syncthreads();
  }
  if (tid == 0) {
    counters->granted = carry_s;
    counters->alive += carry_s;
  }
}

// Writes yd_grant records and creates the TaskDesc of every grant (cc:126-135).
__global__ void __launch_bounds__(1024) k_final_write(const uint32_t* __restrict__ res,
                                                      const yd_task_req* __restrict__ reqs,
                                                      const DynParams* __restrict__ dp,
                                                      const uint32_t* __restrict__ block_off,
                                                      const uint32_t* __restrict__ comp_sv, TaskRing ring,
                                                      yd_grant* __restrict__ out,
                                                      const uint32_t* __restrict__ abort_flag,
                                                      uint32_t* __restrict__ run,
                                                      unsigned long long* __restrict__ ever) {
  if (abort_flag && *abort_flag) return;
  const uint32_t n = dp->n;
  const long long now_ns = dp->now_ns;
  ring.next = dp->ring_next;  // pointers and mask come by value; the window bounds are per call
  __shared__ uint32_t warp_cnt[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t q = blockIdx.x * 1024 + tid;
  uint32_t r = q < n ? res[q] : kResEnvNotFound;
  bool granted = r < kResTimeout;
  if (granted) r = comp_sv[r];  // solver results index the component-ordered servant list
  uint32_t bal = __ballot_sync(0xffffffffu, granted);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  uint32_t before = 0;
  for (uint32_t w = 0; w < warp; ++w) before += warp_cnt[w];
  before += __popc(bal & ((1u << lane) - 1));
  if (q >= n) return;
  uint4 g;  // {task_id lo, task_id hi, servant_index, status} == yd_grant
  if (granted) {
    uint64_t id = ring.next + block_off[blockIdx.x] + before;
    const unsigned long long xid = ring.ext(id);
    g = make_uint4((uint32_t)xid, (uint32_t)(xid >> 32), r, YD_STATUS_GRANTED);
    uint64_t slot = id & ring.mask;
    const yd_task_req rq = reqs[q];
    ring.exp[slot] = now_ns + rq.expires_in_ns;
    ring.srv[slot] = r;
    ring.flags[slot] = kTaskAlive | ((rq.flags & YD_REQ_FLAG_PREFETCH) ? kTaskPrefetch : 0u);
    if (run) {  // ++running_tasks, ++ever_assigned_tasks (cc:123-124); the slot-stream solvers leave it to us
      atomicAdd(&run[r], 1u);
      atomicAdd(&ever[r], 1ull);
    }
  } else {
    g = make_uint4(0u, 0u, YD_NO_SERVANT,
                   (r == kResTimeout) ? YD_STATUS_TIMEOUT : YD_STATUS_ENVIRONMENT_NOT_FOUND);
  }
  *reinterpret_cast<uint4*>(out + q) = g;  // one 16-byte store
}

// The three kernels above in ONE launch: task ids are the FIFO ordinals of the grants, i.e. an exclusive prefix over
// the per-block grant counts -- here a single-pass scan with decoupled look-back: a block takes a ticket (so that its
// predecessors are running or done), publishes its count, sums its predecessors' published counts back to the nearest
// one that already knows its inclusive prefix, and publishes its own.  `look` = one zeroed 64-bit word per block
// (bits 63..62: 1 = count, 2 = inclusive prefix; low bits: the value) + the ticket counter behind them.
//
// final_tile: tile `vb` of 1024 requests, r = the solver's verdict for request vb * 1024 + tid (kResEnvNotFound beyond
// the queue's end).  Tiles below vb must be running or done.  kPacked: 8-byte grants {servant_index, status << 30 |
// FIFO ordinal of the grant}, see yd_grant8 in ydsched.h.
// kPos: r is already a registry position (else an index into comp_sv).  kBase: the caller knows the grants of the tiles
// before this one (`base`; the fused solo kernel derives it from its per-class counts): no look-back, `look` is unused.
// kLease: the caller has read the request's lease fields already (`lflags`, `lexp`: ReqView::lease), so that their load
// overlaps its own; else they are read here, once the grant is known.  kCount: ++running_tasks and ++ever of the
// granted servant, one atomic each per grant (the speculative solo solve counts them per servant instead, fused.cuh).
template <bool kPacked, bool kPos = false, bool kBase = false, bool kLease = false, bool kCount = true>
__device__ __forceinline__ void final_tile(uint32_t vb, uint32_t last_vb, uint32_t r, uint32_t n, long long now_ns,
                                           const ReqView& reqs, unsigned long long* __restrict__ look,
                                           const uint32_t* __restrict__ comp_sv, const TaskRing& ring,
                                           void* __restrict__ out, Counters* __restrict__ counters,
                                           uint32_t* __restrict__ run, unsigned long long* __restrict__ ever,
                                           unsigned long long base = 0, uint32_t lflags = 0, long long lexp = 0) {
  __shared__ uint32_t warp_cnt[32];
  __shared__ unsigned long long s_excl;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t q = vb * 1024 + tid;
  const bool granted = r < kResTimeout;
  if (granted && !kPos) r = comp_sv[r];  // solver results index the component-ordered servant list
  const uint32_t bal = __ballot_sync(0xffffffffu, granted);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  // every warp scans the 32 warp counts itself: its grants in the lower warps, and the tile's
  uint32_t wpre = warp_cnt[lane];
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, wpre, d);
    if (lane >= d) wpre += y;
  }
  const uint32_t mine = __shfl_sync(0xffffffffu, wpre, 31);
  wpre = __shfl_sync(0xffffffffu, wpre, (warp + 31) & 31);
  if (warp == 0) wpre = 0;
  if (kBase) {  // the caller knows the tiles before this one: no look-back, no second barrier
    if (warp == 0 && lane == 0 && vb == last_vb) {  // the last block knows the batch's total
      counters->granted = base + mine;
      counters->alive += base + mine;
    }
  } else if (warp == 0) {
    volatile unsigned long long* vl = look;
    if (lane == 0) { __threadfence(); vl[vb] = (1ull << 62) | mine; }
    unsigned long long excl = 0ull;
    int at = (int)vb - 1;
    while (at >= 0) {
      const int idx = at - (int)lane;
      unsigned long long v;
      do {
        v = idx >= 0 ? vl[idx] : (2ull << 62);  // before the first block: an inclusive prefix of zero
      } while (__any_sync(0xffffffffu, (v >> 62) == 0));
      const uint32_t incl = __ballot_sync(0xffffffffu, (v >> 62) == 2);
      const unsigned long long val = v & ((1ull << 62) - 1);
      if (incl) {
        const uint32_t first = __ffs(incl) - 1;  // the nearest predecessor that knows its inclusive prefix
        unsigned long long part = lane <= first ? val : 0ull;
#pragma unroll
        for (int d = 16; d; d >>= 1) part += __shfl_xor_sync(0xffffffffu, part, d);
        excl += part;
        break;
      }
      unsigned long long part = val;
#pragma unroll
      for (int d = 16; d; d >>= 1) part += __shfl_xor_sync(0xffffffffu, part, d);
      excl += part;
      at -= 32;
    }
    if (lane == 0) {
      __threadfence();
      vl[vb] = (2ull << 62) | (excl + mine);
      s_excl = excl;
      if (vb == last_vb) {  // the last block knows the batch's total
        counters->granted = excl + mine;
        counters->alive += excl + mine;
      }
    }
  }
  if (!kBase) __syncthreads();
  if (q < n) {
    const uint32_t before = wpre + __popc(bal & ((1u << lane) - 1));
    const uint64_t ordinal = (kBase ? base : s_excl) + before;
    uint32_t status;
    if (granted) {
      status = YD_STATUS_GRANTED;
      const uint64_t id = ring.next + ordinal;
      const uint64_t slot = id & ring.mask;
      uint32_t rflags = lflags;
      long long expires_in_ns = lexp;
      if (!kLease) reqs.lease(q, rflags, expires_in_ns);
      ring.exp[slot] = now_ns + expires_in_ns;
      ring.srv[slot] = r;
      ring.flags[slot] = kTaskAlive | ((rflags & YD_REQ_FLAG_PREFETCH) ? kTaskPrefetch : 0u);
      if (kCount) {
        atomicAdd(&run[r], 1u);  // ++running_tasks, ++ever_assigned_tasks (cc:123-124)
        atomicAdd(&ever[r], 1ull);
      }
    } else {
      status = (r == kResTimeout) ? YD_STATUS_TIMEOUT : YD_STATUS_ENVIRONMENT_NOT_FOUND;
      r = YD_NO_SERVANT;
    }
    if (kPacked) {
      reinterpret_cast<uint2*>(out)[q] = make_uint2(r, (status << 30) | (granted ? (uint32_t)ordinal : 0u));
    } else {
      const unsigned long long xid = granted ? ring.ext(ring.next + ordinal) : 0ull;
      // {task_id lo, task_id hi, servant_index, status} == yd_grant, one 16-byte store
      reinterpret_cast<uint4*>(out)[q] = make_uint4((uint32_t)xid, (uint32_t)(xid >> 32), r, status);
    }
  }
  __syncthreads();  // (warp_cnt / s_excl are reused when a block handles several tiles)
}

__global__ void __launch_bounds__(1024) k_final_fused(const uint32_t* __restrict__ res,
                                                      const yd_task_req* __restrict__ reqs,
                                                      const DynParams* __restrict__ dp,
                                                      unsigned long long* __restrict__ look, uint32_t nb,
                                                      const uint32_t* __restrict__ comp_sv, TaskRing ring,
                                                      yd_grant* __restrict__ out, Counters* __restrict__ counters,
                                                      const uint32_t* __restrict__ abort_flag,
                                                      uint32_t* __restrict__ run, unsigned long long* __restrict__ ever) {
  if (abort_flag && *abort_flag) return;
  __shared__ uint32_t s_vb;
  if (threadIdx.x == 0) s_vb = (uint32_t)atomicAdd(&look[nb], 1ull);
  __syncthreads();
  const uint32_t vb = s_vb;
  const uint32_t n = dp->n;
  ring.next = dp->ring_next;
  const uint32_t q = vb * 1024 + threadIdx.x;
  final_tile<false>(vb, nb - 1, q < n ? res[q] : kResEnvNotFound, n, dp->now_ns, ReqView{reqs, nullptr}, look, comp_sv, ring, out, counters,
                    run, ever);
}

// run[] += claims, ever[] += claims: the all-reduced per-servant slot claims of a range-sharded solve.
__global__ void k_apply_claims(uint32_t S, const uint32_t* __restrict__ claims, uint32_t* __restrict__ run,
                               unsigned long long* __restrict__ ever, const uint32_t* __restrict__ abort_flag) {
  if (abort_flag && *abort_flag) return;
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S || claims[s] == 0) return;
  run[s] += claims[s];
  ever[s] += claims[s];
}

// ---- FreeTask (cc:167-188), one thread per id --------------------------------
// `dec` (range-sharded handles only, else null): this rank's running_tasks decrements since the last collective
// call, which hands them to the other ranks (shard_host.inc).  run == null: the lease is forgotten, running_tasks
// stays (a lease another rank holds, shard_host.inc).
__global__ void k_free(const unsigned long long* __restrict__ ids, uint32_t n, TaskRing ring,
                       uint32_t* __restrict__ run, Counters* __restrict__ counters, uint32_t* __restrict__ dec) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long id;
  if (!ring.loc(ids[i], &id) || id < ring.lo || id >= ring.next) return;  // unknown id: FreeTask just returns (cc:175-179)
  uint64_t slot = id & ring.mask;
  uint32_t old = atomicExch(&ring.flags[slot], 0u);  // duplicates in one call: first one wins
  if (old & kTaskAlive) {
    if (run) atomicSub(&run[ring.srv[slot]], 1u);
    if (dec) atomicAdd(&dec[ring.srv[slot]], 1u);
    atomicAdd(&counters->alive, ~0ull);
    if (old & kTaskZombie) atomicAdd(&counters->zombies, ~0ull);
  }
}

// ---- KeepTaskAlive (cc:142-165) ----------------------------------------------
// `ok` is bytes for one handle, u32 words for a range-sharded group (the words travel in a sum all-reduce).
// `lens` == null: every id gets `new_expires_in_ns`.  Otherwise id i gets lens[i], and only the id's last occurrence in
// the array (last[i] != 0, marked by the host) writes the expiry, so that the last length wins as in the loop of single
// calls.  The answer depends on the lease's flags alone, which this kernel does not change: every occurrence gets it.
template <typename Flag>
__global__ void k_keep_alive(const unsigned long long* __restrict__ ids, uint32_t n, long long now_ns,
                             long long new_expires_in_ns, const long long* __restrict__ lens,
                             const uint8_t* __restrict__ last, TaskRing ring, Flag* __restrict__ ok) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long id;
  uint8_t r = 0;
  if (ring.loc(ids[i], &id) && id >= ring.lo && id < ring.next) {
    uint64_t slot = id & ring.mask;
    uint32_t f = ring.flags[slot];
    if ((f & kTaskAlive) && !(f & kTaskZombie)) {
      if (!lens) ring.exp[slot] = now_ns + new_expires_in_ns;
      else if (last[i]) ring.exp[slot] = now_ns + lens[i];
      r = 1;
    }
  }
  ok[i] = r;
}

// ---- OnExpirationTimer (cc:498-536) over the live window ---------------------
// remap: old registry position -> new position, or kNone if the servant expired
// (then the task is an orphan and is forgotten without becoming a zombie,
// cc:478-496).  remap == nullptr when no servant expired.
__global__ void k_tick(TaskRing ring, long long now_ns, const uint32_t* __restrict__ remap,
                       Counters* __restrict__ counters) {
  unsigned long long id = ring.lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long my_min = ~0ull;
  long long d_alive = 0, d_zombie = 0;
  if (id < ring.next) {
    uint64_t slot = id & ring.mask;
    uint32_t f = ring.flags[slot];
    if (f & kTaskAlive) {
      bool gone = false;
      if (remap) {
        uint32_t np = remap[ring.srv[slot]];
        if (np == kNone) {
          ring.flags[slot] = 0;
          gone = true;
          d_alive = -1;
          if (f & kTaskZombie) d_zombie = -1;
        } else {
          ring.srv[slot] = np;
        }
      }
      if (!gone) {
        my_min = id;
        if (!(f & kTaskZombie) && ring.exp[slot] < now_ns) {
          ring.flags[slot] = f | kTaskZombie;
          d_zombie = 1;
        }
      }
    }
  }
  // block reduction, then one atomic per block per counter
  __shared__ unsigned long long s_min[32];
  __shared__ int s_a[32], s_z[32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int a = (int)d_alive, z = (int)d_zombie;
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    unsigned long long o = __shfl_xor_sync(0xffffffffu, my_min, d);
    my_min = o < my_min ? o : my_min;
    a += __shfl_xor_sync(0xffffffffu, a, d);
    z += __shfl_xor_sync(0xffffffffu, z, d);
  }
  if (lane == 0) { s_min[warp] = my_min; s_a[warp] = a; s_z[warp] = z; }
  __syncthreads();
  if (warp == 0) {
    uint32_t nw = blockDim.x >> 5;
    my_min = lane < nw ? s_min[lane] : ~0ull;
    a = lane < nw ? s_a[lane] : 0;
    z = lane < nw ? s_z[lane] : 0;
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      unsigned long long o = __shfl_xor_sync(0xffffffffu, my_min, d);
      my_min = o < my_min ? o : my_min;
      a += __shfl_xor_sync(0xffffffffu, a, d);
      z += __shfl_xor_sync(0xffffffffu, z, d);
    }
    if (lane == 0) {
      if (my_min != ~0ull) atomicMin(&counters->min_live, my_min);
      if (a) atomicAdd(&counters->alive, (unsigned long long)(long long)a);
      if (z) atomicAdd(&counters->zombies, (unsigned long long)(long long)z);
    }
  }
}

// Order-preserving erase of expired servants from the state arrays (cc:503-516).
__global__ void k_compact_servants(uint32_t S_old, const uint32_t* __restrict__ remap,
                                   const uint32_t* __restrict__ run_old,
                                   const unsigned long long* __restrict__ ever_old,
                                   uint32_t* __restrict__ run_new,
                                   unsigned long long* __restrict__ ever_new,
                                   const uint32_t* __restrict__ dec_old, uint32_t* __restrict__ dec_new) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S_old) return;
  uint32_t np = remap[s];
  if (np != kNone) {
    run_new[np] = run_old[s];
    ever_new[np] = ever_old[s];
    if (dec_new) dec_new[np] = dec_old[s];
  }
}

// ---- NotifyServantRunningTasks (cc:222-277), any number of servants per launch ---------------
// One heartbeat = (registry position, the task ids the servant reports).  The host sorts the
// heartbeats of a batch by position: item_pos[] ascending, item_off[] the CSR offsets into ids[].
struct NotifyBatch {
  const uint32_t* item_pos;            // [n_items] ascending, distinct
  const uint32_t* item_off;            // [n_items + 1]
  const unsigned long long* ids;       // [item_off[n_items]] reported task_grant_ids
  uint32_t n_items;
};

__device__ __forceinline__ uint32_t notify_find_item(const NotifyBatch& b, uint32_t pos) {
  uint32_t lo = 0, hi = b.n_items;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint32_t p = b.item_pos[mid];
    if (p == pos) return mid;
    if (p < pos) lo = mid + 1; else hi = mid;
  }
  return kNone;
}

// Sweep: zombies of a heartbeating servant that the servant no longer reports are freed
// (UnsafeSweepZombiesOf, cc:453-476).  One thread per lease of the live window; zombies are rare,
// so the scan of the servant's reported ids (global memory, any length) is off the common path.  `dec` as in k_free.
__global__ void k_notify_sweep(TaskRing ring, NotifyBatch b, uint32_t* __restrict__ run,
                               Counters* __restrict__ counters, uint32_t* __restrict__ dec) {
  unsigned long long id = ring.lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= ring.next) return;
  uint64_t slot = id & ring.mask;
  uint32_t f = ring.flags[slot];
  if ((f & (kTaskAlive | kTaskZombie)) != (kTaskAlive | kTaskZombie)) return;
  const uint32_t pos = ring.srv[slot];
  const uint32_t item = notify_find_item(b, pos);
  if (item == kNone) return;  // that servant did not heartbeat in this batch
  const unsigned long long xid = ring.ext(id);
  for (uint32_t i = b.item_off[item], e = b.item_off[item + 1]; i < e; ++i) {
    if (b.ids[i] == xid) return;  // still reported: stays a zombie
  }
  ring.flags[slot] = 0;
  atomicSub(&run[pos], 1u);
  if (dec) atomicAdd(&dec[pos], 1u);
  atomicAdd(&counters->alive, ~0ull);
  atomicAdd(&counters->zombies, ~0ull);
}

// Check: a reported id is "permitted" iff it is a live, non-zombie grant on the reporting
// servant (cc:257-262); everything else goes back to the daemon as unknown.  One thread per id.  A permitted id gets
// `tag`: 1 in bytes for one handle; rank + 1 in u32 words for a range-sharded group, whose sum over the ranks then says
// both whether and where the lease lives (it lives on one rank at most).
template <typename Flag>
__global__ void k_notify_check(TaskRing ring, NotifyBatch b, uint32_t n_ids, Flag* __restrict__ permitted, Flag tag) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ids) return;
  uint32_t lo = 0, hi = b.n_items;  // the item whose id range holds i
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (b.item_off[mid] <= i) lo = mid; else hi = mid;
  }
  const uint32_t pos = b.item_pos[lo];
  unsigned long long id;
  uint8_t ok = 0;
  if (ring.loc(b.ids[i], &id) && id >= ring.lo && id < ring.next) {
    uint64_t slot = id & ring.mask;
    uint32_t f = ring.flags[slot];
    ok = (f & kTaskAlive) && !(f & kTaskZombie) && ring.srv[slot] == pos;
  }
  permitted[i] = ok ? tag : Flag(0);
}

// Ring growth: re-place the live window into a ring twice (or more) the size.
__global__ void k_ring_grow(TaskRing old_ring, TaskRing new_ring) {
  unsigned long long id = old_ring.lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= old_ring.next) return;
  uint64_t so = id & old_ring.mask, sn = id & new_ring.mask;
  new_ring.exp[sn] = old_ring.exp[so];
  new_ring.srv[sn] = old_ring.srv[so];
  new_ring.flags[sn] = old_ring.flags[so];
}

}  // namespace yd
