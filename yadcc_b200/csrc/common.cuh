// common.cuh -- shared definitions for the sm_90a scheduler kernels.
//
// HBM layout (all arrays are structure-of-arrays, indexed by REGISTRY POSITION,
// i.e. the reference's `servants_.servants` vector index, whose order is the
// pick tie-break; task_dispatcher.h:195-197, .cc:444):
//
//   servant facts   nproc[S] load[S] max_tasks[S] flags[S] version[S]   (u32/i32, rewritten on heartbeat)
//   servant state   run[S] (u32 running_tasks)  ever[S] (u64 ever_assigned_tasks)
//   lease ring      t_exp[C] (i64 ns) t_srv[C] (u32 position) t_flags[C] (u32)
//                   slot of task id = id & (C-1); window [lo, next) of ids is live-or-dead,
//                   everything below lo is dead (TaskRegistry, task_dispatcher.h:217-220)
//   per solve       reqs[n] (24 B AoS, as received)  res[n] (u32)  grants[n] (16 B AoS)
//                   slot codes: one u32 per (servant, running_tasks value) -- the
//                   (task x servant) cost-matrix column for that servant, see slots.cuh
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "ydsched.h"

namespace yd {

constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kFull = 0xFFFFFFFFu;            // slot code of a servant that is not free
constexpr uint32_t kResEnvNotFound = 0xFFFFFFFFu;  // res[] encodings (anything below is a position)
constexpr uint32_t kResTimeout = 0xFFFFFFFEu;
constexpr uint32_t kSelfBit = 0x80000000u;  // "tier 2": the requestor's own servant, last resort
constexpr uint32_t kTierBit = 0x40000000u;  // tier 1: not (dedicated and below 50% of its cores)
constexpr int kFracBits = 27;

// Largest capacity for which floor(r * 2^27 / cap) orders r/cap exactly like the
// reference's double division (distinct fractions with denominators <= 2^13
// differ by >= 2^-26 > 2^-27, and equal fractions give equal floors).  Above it
// the wide (64-bit key) path is used.
constexpr uint32_t kNarrowCapLimit = 8192;

constexpr uint32_t kFlagDedicated = 1u;  // ServantPriority == DEDICATED
constexpr uint32_t kFlagLowMem = 2u;     // total_memory != 0 && available < min_memory (cc:286-292)

constexpr uint32_t kTaskAlive = 1u;
constexpr uint32_t kTaskZombie = 2u;
constexpr uint32_t kTaskPrefetch = 4u;

struct Counters {
  unsigned long long granted;   // grants of the last solve
  unsigned long long alive;     // live leases (zombies included)
  unsigned long long zombies;   // live leases marked zombie
  unsigned long long min_live;  // smallest live id seen by the last tick (or ~0)
  unsigned long long slots;     // slot-table entries of the last solve
  unsigned long long spare;
  unsigned long long pad[4];    // solver diagnostics (see solve_stream.cuh)
};

// Per-call scalars.  They live in device memory (copied from a pinned host struct by the
// first node of the captured solve graph) so that one CUDA graph replays for every call
// of the same size class.
struct DynParams {
  uint32_t n;  // exact number of requests (grids are sized for the next power of two)
  uint32_t slot_clamp;  // no servant needs more slots than the batch has requests: n on one GPU, the whole
                        // queue's length (or "no limit") when the queue is sharded over ranks
  long long now_ns;
  unsigned long long ring_lo, ring_next;
};

// Where the per-class FIFO request records of the merge solver live, and how this rank's piece of
// the queue fits into the whole (one GPU: the whole queue is this rank's).  Filled by k_rq_layout.
struct RqLayout {
  uint32_t* goff;    // [classes] requests of the class on LOWER ranks (0 on one GPU)
  uint32_t* gn;      // [classes] requests of the class in the whole queue
  uint32_t* win;     // [classes] how many of them have a record in rq: global class ranks [0, win)
  uint32_t* base;    // [classes] first record of the class in rq
  uint32_t* total;   // [1] records in rq
  uint32_t q_base;   // global queue index of this rank's first request
  uint32_t n_local;  // requests this rank holds (bounds res[] writes; exact value, not the grid bound)
  uint32_t sharded;  // 1: the queue is range-sharded over several ranks (shard.cuh); 0: the four arrays above are not
                     //    used, the layout is the FIFO rank scan itself (class c's records start where its ranks do)
  const uint32_t* rank_off;  // scanned (class-major, tile-minor) request counts of this rank
  uint32_t nrt;              // tiles per class row
  __device__ __forceinline__ uint32_t Goff(uint32_t c) const { return sharded ? goff[c] : 0u; }
  __device__ __forceinline__ uint32_t Gn(uint32_t c) const { return sharded ? gn[c] : rank_off[(c + 1) * nrt] - rank_off[c * nrt]; }
  __device__ __forceinline__ uint32_t Win(uint32_t c) const { return sharded ? win[c] : Gn(c); }
  __device__ __forceinline__ uint32_t Base(uint32_t c) const { return sharded ? base[c] : rank_off[c * nrt]; }
};

// The request queue as the kernels read it: the 24-byte records of the C ABI (yd_task_req), or -- inside the one kernel
// that receives a packed upload (fused.cuh) -- the 16-byte records of yd_task_req16: {env_id, min_version,
// requestor_ip, lease} with lease = expires_in_ms | prefetch << 31 (the RPC surface counts leases in milliseconds,
// scheduler.proto next_keep_alive_in_ms).
struct ReqView {
  const yd_task_req* r24;
  const uint4* r16;  // null: read r24
  __device__ __forceinline__ void head(uint32_t q, uint32_t& env, uint32_t& mv) const {
    const uint2 w = r16 ? reinterpret_cast<const uint2*>(r16 + q)[0] : reinterpret_cast<const uint2*>(r24 + q)[0];
    env = w.x; mv = w.y;
  }
  __device__ __forceinline__ uint32_t ip(uint32_t q) const {
    return r16 ? reinterpret_cast<const uint2*>(r16 + q)[1].x : reinterpret_cast<const uint2*>(r24 + q)[1].x;
  }
  __device__ __forceinline__ void lease(uint32_t q, uint32_t& flags, long long& expires_in_ns) const {
    if (r16) {
      const uint32_t w = reinterpret_cast<const uint2*>(r16 + q)[1].y;
      flags = (w >> 31) ? YD_REQ_FLAG_PREFETCH : 0u;
      expires_in_ns = (long long)(w & 0x7fffffffu) * 1000000ll;
    } else {
      flags = reinterpret_cast<const uint2*>(r24 + q)[1].y;
      expires_in_ns = reinterpret_cast<const long long*>(r24 + q)[2];
    }
  }
};

struct ServantArrays {
  uint32_t* nproc;
  uint32_t* load;
  uint32_t* max_tasks;
  uint32_t* flags;
  int32_t* version;
  uint32_t* run;
  unsigned long long* ever;
};

struct TaskRing {
  long long* exp;
  uint32_t* srv;
  uint32_t* flags;
  uint64_t mask;  // capacity - 1
  uint64_t lo;    // LOCAL ids below lo are dead
  uint64_t next;  // next LOCAL id to hand out
  // external id = local * id_stride + id_offset (sharded deployments; 1 / 0 otherwise)
  uint32_t id_stride, id_offset;
  __host__ __device__ unsigned long long ext(unsigned long long local) const { return local * id_stride + id_offset; }
  // external -> local; false if the id cannot be one of ours
  __host__ __device__ bool loc(unsigned long long external, unsigned long long* local) const {
    if (external < id_offset) return false;
    const unsigned long long d = external - id_offset;
    if (id_stride > 1 && d % id_stride) return false;
    *local = id_stride > 1 ? d / id_stride : d;
    return true;
  }
};

// GetCapacityAvailable (task_dispatcher.cc:283-313) for the not-low-memory case,
// as a function of running_tasks r.  All operands are zero-extended u32, so the
// reference's size_t/int64 juggling is plain signed arithmetic here.
__host__ __device__ inline int64_t capacity_at(uint32_t max_tasks, uint32_t nproc, uint32_t load,
                                               uint64_t r) {
  int64_t foreign = (int64_t)load - (int64_t)r;
  if (foreign < 0) foreign = 0;
  int64_t avail = (int64_t)nproc - foreign;
  if (avail < 0) avail = 0;
  return avail < (int64_t)max_tasks ? avail : (int64_t)max_tasks;
}

// First running_tasks value at which the servant is no longer free
// (`running_tasks >= GetCapacityAvailable`, cc:353).  Derivation in DESIGN.md:
// with P = nproc, L = load, M = max_tasks the servant is free at r iff
// !lowmem && P > L && r < min(M, P).
__host__ __device__ inline uint32_t free_end(uint32_t max_tasks, uint32_t nproc, uint32_t load,
                                             uint32_t flags) {
  if ((flags & kFlagLowMem) || nproc <= load) return 0;
  return max_tasks < nproc ? max_tasks : nproc;
}

// Lowercase hex of the four bytes of x (byte 0 first), as 8 characters in a little-endian word: the form in which a
// delegate's keys carry a 32-byte digest (ydsched.h, yd_prefilter_packed).
__device__ __forceinline__ unsigned long long hex_u32(uint32_t x) {
  unsigned long long n = 0;  // one nibble per byte, the high nibble of each input byte first
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    n |= (unsigned long long)((x >> (8 * b + 4)) & 15u) << (16 * b);
    n |= (unsigned long long)((x >> (8 * b)) & 15u) << (16 * b + 8);
  }
  // '0' + n, and 'a' - '0' - 10 = 39 more where n > 9 (n + 6 carries into bit 4 of its byte exactly then)
  return n + 0x3030303030303030ull + (((n + 0x0606060606060606ull) >> 4) & 0x0101010101010101ull) * 39u;
}

// The 32-byte digest record `d` (16-byte aligned) as 8 words of its 64-character hex: h[k] = characters 8k .. 8k+7.
__device__ __forceinline__ void hex_digest(const unsigned char* __restrict__ d, unsigned long long h[8]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(d)), b = __ldg(reinterpret_cast<const uint4*>(d) + 1);
  h[0] = hex_u32(a.x); h[1] = hex_u32(a.y); h[2] = hex_u32(a.z); h[3] = hex_u32(a.w);
  h[4] = hex_u32(b.x); h[5] = hex_u32(b.y); h[6] = hex_u32(b.z); h[7] = hex_u32(b.w);
}

}  // namespace yd

#define YD_CUDA_CHECK(expr)                                                                   \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      fprintf(stderr, "ydsched: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e__), __FILE__, \
              __LINE__, cudaGetErrorString(e__));                                             \
      abort();                                                                                \
    }                                                                                         \
  } while (0)
