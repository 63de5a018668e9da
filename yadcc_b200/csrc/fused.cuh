// fused.cuh -- the front of the slot-stream pipeline as ONE persistent kernel.
//
// At the headline size (100 k requests x 2 k servants) every kernel of the pipeline in ydsched.cu:LaunchStream does a
// few microseconds of work and costs a few more to launch and drain: ten dependent kernels are ten launch latencies
// (the kernel-by-kernel pipeline is 13 kernels per solve).  Here the same
// device functions (classes.cuh, parallel.cuh, tasks.cuh) run as phases of one co-resident grid -- one block of 1024
// threads per SM, tiles handed out round-robin -- separated by grid barriers:
//
//   P1  class table insert of every request                       (cls_insert_one; unpacks a 16-byte upload)
//   E1  barrier; the LAST block to arrive numbers the classes and picks the solver modes (cls_finalize_block)
//   P3  per-tile FIFO rank counts, per-tile list membership ballots + counts, per-class eligible counts
//   E2  barrier; the last block to arrive scans both (class, tile) count matrices
//   P5  per-class sorted slot lists                                 (list_fill_tile)
//   B3  barrier
//   P6  verdicts of the data-parallel components, FIFO records of the merge components (rank_assign_one) and --
//       `solo`, when every component with requests is data-parallel -- task ids (in closed form from the per-class
//       counts, see fused_class_grants), grants, leases, ++running_tasks (final_tile): the whole solve in one launch.
//
// Not solo: res[] goes to HBM and the merge / sequential solvers and k_final_fused follow as separate launches.
// A solo kernel that finds a component it cannot decide raises flag 4 and decides nothing; the host replays the batch
// with the general sequence (and remembers which one the workload needs).
//
// E1 only numbers the classes, and a scheduler's class set -- (digest, min_version) pairs -- rarely changes from one
// batch to the next.  So a solo solve whose class set is the one of the previous solo solve KEEPS its class table (keys,
// slot_cls, cls_env / mv / comp, meta, comp_mode) and writes it out per digest and per servant (kept_env, kept_sv), and
// the next solo solve runs SPECULATIVELY on it, with one barrier:
//
//   A   every request looked up in the kept table (kept_class: the digest's kept_env word and the IP's component mask,
//       two independent loads) and ranked in its tile (rank_in_tile): its class and rank stay in registers, as tile t is
//       handled by block t % G in both phases; list ballots and counts, one list per slot at most
//       (list_count_tile_kept); eligible servants per class (servant versions and max_tasks change without a new
//       topology)
//   --  barrier
//   B   P6 as above (the lite selection, closed-form task ids), without the per-grant running_tasks / ever atomics:
//       each servant's grants are counted once, by one warp, in blocks without a request tile
//       (fused_servant_counters).  The last block resets the barrier words, nothing else.
//
// A request MISSES when its digest is held by a component but its class is not in the table, or when its IP is that of
// a servant of its component: flag kFlagSpecMiss, nothing is decided, the last block clears the scratch (the kept table
// too) and the host replays the batch without speculation.  Why a hit decides exactly what a full solve decides: a kept
// table was written by a completed solo solve, so each of its components holds one class and is data-parallel.  If
// every request hits and none comes from a servant of its component, each component with requests still has exactly
// that one class and no self-request, and cls_finalize_block would pick the same modes; a kept class without requests
// only makes a component without requests, which decides nothing (and grants nothing: min(0, L) = 0).  Class ids do not
// enter decisions: ranks and lists are per class.
//
// The barrier is the cooperative-groups pattern (bar.sync; one thread: fence, atomic arrive, spin, fence; bar.sync).  The
// grid never exceeds the number of SMs, so all blocks are resident; a block that has to wait for other kernels to drain
// first only delays the barrier.
#pragma once
#include "parallel.cuh"
#include <cstddef>
#include "tasks.cuh"

namespace yd {

// The per-call scalars.  A solo solve is ONE plain kernel launch and gets them by value (kernel parameters); the graphed
// general sequence reads them from HBM, where the graph's first node copies them.  (They are NOT read from mapped host
// memory: a dependent load over PCIe at the top of the kernel cost ~70 us apiece on the measured boxes.)
struct FusedScalars {
  DynParams dyn;
  unsigned long long seq;  // launch counter, echoed in the report
  // Zero-copy I/O, when the caller's arrays are page-locked (yd_alloc_host): device-visible addresses of the caller's
  // request array (read once, by the first phase, which leaves a copy in HBM for the later ones) and grant array
  // (written by the last phase of a solo solve) -- no copy-engine transfer before or after the kernel.  Else null.
  const void* zc_in;
  void* zc_out;
  // Solo, not speculative: the class-set fingerprint of the previous such solve (0: none).  A solve that finds the same
  // class set again keeps its class table for the speculative variant; any other leaves the scratch clean.
  unsigned long long kept_fp;
};

// The solo kernel's result, in MAPPED pinned host memory (posted writes; the host reads it after the stream has drained):
// no copy node after the kernel either.
struct FusedHostIO {
  unsigned long long done_seq;   // = the launch's seq once the record below is complete (written last)
  unsigned long long granted;    // grants of the batch
  uint32_t meta[8];              // the class table's meta words (meta[1] != 0: nothing was decided, see ClassTable)
  unsigned long long classes_fp; // solo, not speculative: fingerprint of the batch's class set (fused_classes_fp)
};

// Flag (meta[1]) of a speculative solve that met a request the kept class table cannot decide: nothing was decided, the
// scratch is clean, the host replays the batch without speculation.
constexpr uint32_t kFlagSpecMiss = 5;

// What a completed solo solve keeps of its class table for the next, speculative one: the keys (behind res[]), comp_mode,
// and the head of the class region (MakeClassTable's layout): slot_cls, meta, cls_env, cls_mv, cls_comp.
constexpr uint32_t kKeptClsWords = kClsTableSize + 8 + 3 * kMaxClasses;
static_assert(kKeptClsWords % 4 == 0, "the scratch behind the kept words is cleared in 16-byte words");

struct FusedArgs {
  FusedScalars sc;              // by value ...
  const FusedScalars* sc_dev;   // ... or, if not null, in HBM
  FusedHostIO* hio;         // device-side address of the mapped result record (solo)
  DynParams* dyn_out;       // device copy of the scalars for the kernels that follow (not solo)
  unsigned long long* clean_keys;  // solo: what the last block re-initialises for the next solve: the class-table keys ...
  uint4* clean_zero;               // ... and the zeroed scratch region
  uint32_t clean_zero_vec;         //     (16-byte words)
  const yd_task_req* reqs;  // the 24-byte queue in HBM
  yd_task_req* reqs_w;      // packed upload, not solo: the 24-byte records are written here for the kernels that follow
  const uint4* reqs16;      // packed upload (yd_task_req16), or null
  uint4* reqs16_w;          // where a zero-copy read of packed requests leaves its HBM copy (= reqs16)
  TopoView t;
  ClassTable ct;
  ServantArrays sv;
  SlotDecode dec;
  const unsigned long long* m_ptr;  // slots in the kept order
  uint32_t* comp_mode;
  uint32_t n_comps;
  uint32_t n_rtiles, n_ltiles;  // row strides of the two count matrices (sized for the batch's / slot table's size class)
  uint32_t* rcls;
  uint32_t* rrank;
  uint32_t* rself;
  uint32_t* rank_cnt;
  uint32_t* list_cnt;
  uint32_t* list_bal;
  uint32_t* members;  // solo: the per-tile member lists (classes.cuh: list_member_index)
  uint2* list;
  uint32_t list_cap;
  uint2* rq;
  uint32_t* res;
  RqLayout L;
  uint32_t* bar;  // [3], zeroed per solve: arrivals, release epoch, blocks that are done
  // solo
  uint32_t solo, packed_out;
  const uint32_t* comp_sv;
  TaskRing ring;
  void* out;
  Counters* counters;
  uint32_t n_servants;
  uint32_t loff_cache_words;  // solo: dynamic shared memory of the launch, in words; not 0: no leader scans -- every block
                              // derives the list offsets it needs from the raw counts (the host sizes it when they fit)
  uint32_t spec;              // solo, speculative: the class table kept from the last solo solve, one grid barrier
  uint4* kept_env;            // [n_envs] the kept class table per digest (classes.cuh: kept_class) ...
  uint32_t* kept_sv;          // [n_servants] ... and per servant (list_count_tile_kept); both written with the table
  const uint32_t* slot_spos;  // the kept order's sorted position of every row slot (k_slot_records)
  unsigned long long* prof;  // debug (YDSCHED_FUSED_PROF): %globaltimer stamps (kProfHead / kProfBlockWords), else null
};

// YDSCHED_FUSED_PROF: block 0 stamps every phase boundary into prof[0 .. 9).  The speculative variant also stamps, per
// block b, prof[kProfHead + b * kProfBlockWords + k]: k = 0 start, 1..3 end of its first three items of phase A, 4
// barrier arrival, 5 departure, 6 end of phase B; word 7 = the kinds of those items (4 bits each, FusedItem) | the
// number of items << 16; then, for the block's first request tile of phase B, 8 end of the table build (list offsets,
// request prefixes, base), 9 end of the selection, 10 end of final_tile; word 11 = end of the servant counters
// (fused_servant_counters), in the blocks that count them.
constexpr uint32_t kProfHead = 16;
constexpr uint32_t kProfBlockWords = 12;
constexpr uint32_t kProfMaxItems = 3;
enum FusedItem : uint32_t { kItemRequests = 1, kItemSlots = 2, kItemClass = 3 };

__device__ __forceinline__ unsigned long long fused_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void fused_stamp(const FusedArgs& a, int k) {
  if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) a.prof[k] = fused_now();
}
__device__ __forceinline__ void fused_bstamp(const FusedArgs& a, uint32_t k, unsigned long long v) {
  if (a.prof && threadIdx.x == 0) a.prof[kProfHead + blockIdx.x * kProfBlockWords + k] = v;
}

// Pull a table into L2 while the first phase streams the requests: the bench flushes L2 between solves and a scheduler
// that has been idle finds it cold too; the later phases chase indices through these tables and would pay one DRAM
// round trip per dependent load.  One 128-byte line per thread and step, spread over the whole grid.
__device__ __forceinline__ void fused_prefetch(const void* p, size_t bytes) {
  const char* base = static_cast<const char*>(p);
  for (size_t off = (size_t(blockIdx.x) * 1024 + threadIdx.x) * 128; off < bytes; off += size_t(gridDim.x) * 1024 * 128) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(base + off));
  }
}

__device__ __forceinline__ uint32_t fused_atom_add_acq_rel(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ uint32_t fused_ld_acquire(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fused_st_release(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Arrive at barrier episode `epoch` (1, 2, ...).  Returns true in exactly one block: the last one to arrive, which has
// already acquired everybody's writes and must call fused_release after its leader work; the others call fused_wait.
// (bar.sync orders the block's accesses before thread 0's release / after its acquire: the cooperative-groups grid
// barrier with release / acquire accesses instead of full fences.)
__device__ __forceinline__ bool fused_arrive(uint32_t* bar, uint32_t epoch) {
  __shared__ uint32_t s_last;
  __syncthreads();
  if (threadIdx.x == 0) s_last = (fused_atom_add_acq_rel(&bar[0], 1u) + 1 == epoch * gridDim.x) ? 1u : 0u;
  __syncthreads();
  return s_last != 0;
}
__device__ __forceinline__ void fused_release(uint32_t* bar, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x == 0) fused_st_release(&bar[1], epoch);
}
__device__ __forceinline__ void fused_wait(uint32_t* bar, uint32_t epoch) {
  if (threadIdx.x == 0) {
    while (fused_ld_acquire(&bar[1]) < epoch) {}
  }
  __syncthreads();
}
// A barrier without a leader section: arrive, then wait for everybody's arrival (one hop).
__device__ __forceinline__ void fused_barrier(uint32_t* bar, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    fused_atom_add_acq_rel(&bar[0], 1u);
    const uint32_t want = epoch * gridDim.x;
    while (fused_ld_acquire(&bar[0]) < want) {}
  }
  __syncthreads();
}
// The same, with a flag raised by any block delivered with the release: a block that raises it arrives with
// kBarFlag + 1 instead of 1, so the count is the low bits of the word and the flags the high bits; the word each block
// acquires when it leaves holds every block's arrival.  Returns whether any block raised it -- no load after the wait.
constexpr uint32_t kBarFlag = 1u << 24;  // (grids of fewer than 2^24 blocks, fewer than 256 flags)
__device__ __forceinline__ bool fused_barrier_any(uint32_t* bar, uint32_t epoch, bool flag) {
  __shared__ uint32_t s_any;
  const bool mine = __syncthreads_or(flag);
  if (threadIdx.x == 0) {
    fused_atom_add_acq_rel(&bar[0], mine ? kBarFlag + 1u : 1u);
    const uint32_t want = epoch * gridDim.x;
    uint32_t v;
    while (((v = fused_ld_acquire(&bar[0])) & (kBarFlag - 1u)) < want) {}
    s_any = v >> 24;
  }
  __syncthreads();
  return s_any != 0;
}
// "I am done": true in the block that finishes last -- it has acquired everything the grid wrote.
__device__ __forceinline__ bool fused_done_last(uint32_t* bar) {
  __shared__ uint32_t s_fin;
  __syncthreads();
  if (threadIdx.x == 0) s_fin = (fused_atom_add_acq_rel(&bar[2], 1u) + 1 == gridDim.x) ? 1u : 0u;
  __syncthreads();
  return s_fin != 0;
}

// Sum of `v` over the block (1024 threads), returned to every thread.
__device__ __forceinline__ uint32_t fused_block_sum(uint32_t v) {
  __shared__ uint32_t s_part[32];
  const uint32_t lane = threadIdx.x & 31;
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();  // (s_part of the previous call has been read)
  if (lane == 0) s_part[threadIdx.x >> 5] = v;
  __syncthreads();
  return __reduce_add_sync(0xffffffffu, s_part[lane]);
}

// The result record for the host (threads 0..8 of one block): the class table's meta words and the grant count, as
// posted writes into mapped host memory.  The host reads it after the stream has drained, so no ordering is needed
// among the writes.
__device__ __forceinline__ void fused_report(const FusedArgs& a, unsigned long long seq, unsigned long long granted,
                                             unsigned long long fp = 0) {
  FusedHostIO* h = a.hio;
  const uint32_t k = threadIdx.x;
  if (k < 8) h->meta[k] = a.ct.meta[k];
  else if (k == 8) { h->granted = granted; h->classes_fp = fp; h->done_seq = seq; }
}

// Order-independent fingerprint of the class set (the occupied keys of the class table), by one block of 1024 threads:
// the number of classes in the high word, a sum of mixed keys in the low word -- never 0.
__device__ __forceinline__ unsigned long long fused_classes_fp(const unsigned long long* __restrict__ keys) {
  uint32_t cnt = 0, mix = 0;
  for (uint32_t i = threadIdx.x; i < kClsTableSize; i += 1024) {
    const unsigned long long k = keys[i];
    if (k != kClsEmpty) {
      unsigned long long x = k * 0x9e3779b97f4a7c15ull;
      x ^= x >> 31;
      x *= 0xbf58476d1ce4e5b9ull;
      mix += (uint32_t)(x >> 32);
      ++cnt;
    }
  }
  cnt = fused_block_sum(cnt);
  mix = fused_block_sum(mix);
  return ((unsigned long long)(cnt + 1) << 32) | mix;
}

// The kept table per digest (kept_env, classes.cuh) and per servant (kept_sv: the class of its component if it holds
// that class's digest, else kNone), by the one block that keeps the table.  First every digest of a component says "no
// class" and every servant kNone, then each class writes its digest and walks its component's servants.  (Each component
// of a kept table holds one class at most, so nothing is written twice.)
__device__ __forceinline__ void fused_keep_env(const FusedArgs& a) {
  const uint32_t ncls = min(a.ct.meta[0], a.ct.cls_bound);
  for (uint32_t e = threadIdx.x; e < a.t.n_envs; e += 1024) {
    a.kept_env[e] = make_uint4(a.t.env_comp[e] == kNone ? kNone : kKeptNoClass, 0u, 0u, 0u);
  }
  for (uint32_t p = threadIdx.x; p < a.n_servants; p += 1024) a.kept_sv[p] = kNone;
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < ncls; c += 1024) {
    a.kept_env[a.ct.cls_env[c]] = make_uint4(c, a.ct.cls_mv[c], a.ct.cls_comp[c], 0u);
  }
  for (uint32_t c = 0; c < ncls; ++c) {
    const uint32_t comp = a.ct.cls_comp[c], env = a.ct.cls_env[c];
    for (uint32_t i = a.t.comp_sv_off[comp] + threadIdx.x, e = a.t.comp_sv_off[comp + 1]; i < e; i += 1024) {
      const uint32_t pos = a.t.comp_sv[i];
      if (servant_has_env(a.t, pos, env)) a.kept_sv[pos] = c;
    }
  }
}

// In-place exclusive scan of data[0 .. cells) by one block of 1024 threads (8 values per thread and round).
__device__ __forceinline__ void fused_scan_flat(uint32_t* __restrict__ data, uint32_t cells) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t base = 0; base < cells; base += 1024 * 8) {
    const uint32_t i0 = base + tid * 8;
    uint32_t v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (i0 + k < cells) ? data[i0 + k] : 0;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) sum += v[k];
    uint32_t x = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = warp_sums[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const uint32_t carry = carry_s;
    uint32_t run = carry + (warp ? warp_sums[warp - 1] : 0) + x - sum;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (i0 + k < cells) data[i0 + k] = run;
      run += v[k];
    }
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_sums[31];
    __syncthreads();
  }
}

// Solo solves skip the compacted lists: the request of class c (not kNone) with class rank `rank` (its FIFO rank among
// the batch's class-c requests) takes the rank-th member of c's list, found straight from what the count phase left
// behind: class c's (class, tile) offsets (`rows + c * stride`: one word per slot tile + the end, in shared memory when
// they fit) name the slot tile and the rank inside it, and the tile's member list names the servant -- one load.
// `nelig`: the classes' eligible-servant counts.  Returns the verdict: a REGISTRY POSITION, kResTimeout or
// kResEnvNotFound.
__device__ __forceinline__ uint32_t fused_select(uint32_t c, uint32_t rank, const FusedArgs& a,
                                                 const uint32_t* __restrict__ nelig, const uint32_t* __restrict__ rows,
                                                 uint32_t stride) {
  if (nelig[c] == 0) return kResEnvNotFound;  // cc:105-108
  const uint32_t* row = rows + c * stride;
  const uint32_t target = row[0] + rank;
  if (target >= row[a.n_ltiles]) return kResTimeout;  // cc:116-118
  uint32_t lo = 0, hi = a.n_ltiles;                   // the last tile whose offset is <= target holds it
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (row[mid] <= target) lo = mid; else hi = mid;
  }
  return a.members[list_member_index(lo, c, a.ct.cls_bound) + (target - row[lo])] & kMemberPosMask;
}

// Task ids of a solo solve in closed form.  The selection above grants the class-c request with class rank k exactly
// when cls_nelig[c] != 0 && k < L_c (L_c = the length of c's list), so of the `before` class-c requests in the tiles
// before a tile, min(before, L_c) were granted; summed over the classes that is the tile's first FIFO ordinal.  Every
// block derives it from the count matrices it already holds: no tile waits for another.
__device__ __forceinline__ uint32_t fused_class_grants(uint32_t nelig, uint32_t before, uint32_t len) {
  return nelig != 0 ? min(before, len) : 0u;
}

// Speculative solve: ++running_tasks and ++ever_assigned_tasks of every grant, counted per servant instead of two
// atomics per grant in final_tile (on a few hundred lines, which L2 applies one after the other).  The grants of class c
// are the first L'_c = nelig_c ? min(R_c, L_c) : 0 members of its list (R_c requests, L_c members: fused_class_grants),
// and the list is in sorted-slot order.  So servant s, of class c = kept_sv[s] and a version high enough (the test of
// list_count_tile_kept), receives one grant per slot r in [run[s], row_len[s]) whose sorted position (slot_spos) is at
// most that of the list's member at rank L'_c - 1, whose slot the member word names.  One warp per class finds that
// bound, then one warp per servant counts its slots below it and writes run[s] and ever[s] with plain stores: after the
// barrier nothing else reads or writes them.  The servants' facts and the sorted positions of their first 64 free slots
// do not depend on the bounds: they are loaded first, two servants per warp, so that their two round trips overlap the
// two of the bounds (the class rows, then one member word).  `own` / `n_own`: this block's index among the blocks that
// share the servants, and their number.
__device__ __forceinline__ void fused_servant_counters(const FusedArgs& a, uint32_t ncls, uint32_t nb_live, uint32_t own,
                                                       uint32_t n_own) {
  __shared__ uint32_t s_end[kMaxClasses];  // class c grants its list's members at sorted positions below s_end[c]
  __shared__ uint32_t s_mv[kMaxClasses];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t W = n_own * 32, gw = own * 32 + warp;  // this warp's servants: gw + j * W
  uint32_t sc[2], sver[2], srun[2], soff[2], slen[2], sp[2][2];
  unsigned long long sever[2];
  auto fetch = [&](uint32_t s0) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t s = s0 + j * W;
      const bool in = s < a.n_servants;
      sc[j] = in ? a.kept_sv[s] : kNone;
      sver[j] = in ? (uint32_t)a.sv.version[s] : 0u;
      srun[j] = in ? a.sv.run[s] : 0u;
      soff[j] = in ? a.dec.row_off[s] : 0u;
      slen[j] = in ? a.dec.row_len[s] : 0u;
      sever[j] = in ? a.sv.ever[s] : 0ull;
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t r = srun[j] + h * 32 + lane;
        sp[j][h] = sc[j] < ncls && r < slen[j] ? a.slot_spos[soff[j] + r] : kNone;
      }
    }
  };
  fetch(gw);
  for (uint32_t c = warp; c < ncls; c += 32) {
    const uint32_t* rrow = a.rank_cnt + c * a.n_rtiles;
    const uint32_t* lrow = a.list_cnt + c * a.n_ltiles;
    const uint32_t nelig = a.ct.cls_nelig[c], mv = a.ct.cls_mv[c];
    uint32_t R = 0, L = 0;
#pragma unroll 4
    for (uint32_t t = lane; t < nb_live; t += 32) R += rrow[t];
#pragma unroll 4
    for (uint32_t t = lane; t < a.n_ltiles; t += 32) L += lrow[t];
    R = __reduce_add_sync(0xffffffffu, R);
    L = __reduce_add_sync(0xffffffffu, L);
    const uint32_t take = fused_class_grants(nelig, R, L);
    uint32_t end = 0;
    if (take) {  // the slot tile of the member at rank take - 1 (the first whose inclusive prefix exceeds it) and its word
      const uint32_t target = take - 1;
      for (uint32_t t0 = 0, before = 0; t0 < a.n_ltiles; t0 += 32) {
        const uint32_t t = t0 + lane, v = t < a.n_ltiles ? lrow[t] : 0u;
        uint32_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
          if (lane >= d) x += y;
        }
        const uint32_t past = __ballot_sync(0xffffffffu, before + x > target);
        if (past) {
          const uint32_t l = __ffs(past) - 1;
          const uint32_t pre = __shfl_sync(0xffffffffu, before + x - v, l);
          const uint32_t w = a.members[list_member_index(t0 + l, c, a.ct.cls_bound) + (target - pre)];
          end = (t0 + l) * kListTile + (w >> kMemberSlotShift) + 1;
          break;
        }
        before += __shfl_sync(0xffffffffu, x, 31);
      }
    }
    if (lane == 0) { s_end[c] = end; s_mv[c] = mv; }
  }
  __syncthreads();
  for (uint32_t s0 = gw; s0 < a.n_servants; s0 += 2 * W) {
    if (s0 != gw) fetch(s0);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t s = s0 + j * W, c = sc[j];
      if (c >= ncls || sver[j] < s_mv[c] || s_end[c] == 0) continue;  // (the same for the whole warp; kNone beyond S)
      const uint32_t end = s_end[c];
      uint32_t k = (sp[j][0] < end ? 1u : 0u) + (sp[j][1] < end ? 1u : 0u);
      for (uint32_t r = srun[j] + 64 + lane; r < slen[j]; r += 32) k += a.slot_spos[soff[j] + r] < end ? 1u : 0u;
      k = __reduce_add_sync(0xffffffffu, k);
      if (lane == 0 && k) {
        a.sv.run[s] = srun[j] + k;
        a.sv.ever[s] = sever[j] + k;
      }
    }
  }
}

// Blocks that take the servant counters of a speculative solve: those without a request tile when there are at least
// this many, else every block (after its request tiles).
constexpr uint32_t kCounterMinBlocks = 16;

// Request q = tile * 1024 + thread (a block of 1024 threads): its digest id, min_version and requestor IP; false beyond
// the queue's end.  A zero-copy solve first copies the tile from the caller's page-locked array to HBM (every later read
// of the requests, here and in the kernels that follow, hits the copy); a packed upload is also written out as the
// 24-byte records the kernels after this one read (not solo).
__device__ __forceinline__ bool fused_fetch_req(const FusedArgs& a, const ReqView& rv, const char* zc_in, uint32_t tile,
                                                uint32_t n, uint32_t& env, uint32_t& mv, uint32_t& ip) {
  const uint32_t tid = threadIdx.x, q = tile * 1024 + tid;
  if (zc_in) {
    // 16 bytes per thread and step (coalesced reads over PCIe)
    if (a.reqs16) {
      if (q < n) a.reqs16_w[q] = reinterpret_cast<const uint4*>(zc_in)[q];
    } else {
      const uint32_t bytes = min(n - tile * 1024, 1024u) * (uint32_t)sizeof(yd_task_req);  // a multiple of 8
      const char* src = zc_in + size_t(tile) * 1024 * sizeof(yd_task_req);
      char* dst = reinterpret_cast<char*>(const_cast<yd_task_req*>(a.reqs)) + size_t(tile) * 1024 * sizeof(yd_task_req);
      for (uint32_t o = tid * 16; o < bytes; o += 1024 * 16) {
        if (o + 16 <= bytes) *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(src + o);
        else *reinterpret_cast<uint2*>(dst + o) = *reinterpret_cast<const uint2*>(src + o);
      }
    }
    __syncthreads();
  }
  if (q >= n) return false;
  if (a.reqs16) {
    const uint4 w = a.reqs16[q];
    env = w.x; mv = w.y; ip = w.z;
    if (a.reqs_w) {
      uint2* dst = reinterpret_cast<uint2*>(a.reqs_w + q);
      const unsigned long long ns = (unsigned long long)(w.w & 0x7fffffffu) * 1000000ull;
      dst[0] = make_uint2(env, mv);
      dst[1] = make_uint2(ip, (w.w >> 31) ? YD_REQ_FLAG_PREFETCH : 0u);
      dst[2] = make_uint2((uint32_t)ns, (uint32_t)(ns >> 32));
    }
  } else {
    rv.head(q, env, mv);
    ip = rv.ip(q);
  }
  return true;
}

__global__ void __launch_bounds__(1024, 1) k_fused_front(FusedArgs a) {
  extern __shared__ uint32_t s_loff[];  // solo: the scanned list offsets, when a.loff_cache_words holds them
  __shared__ unsigned long long s_seen[64];
  __shared__ DynParams s_dyn;
  __shared__ unsigned long long s_seq, s_zc_in, s_zc_out, s_kept_fp;
  const uint32_t tid = threadIdx.x, G = gridDim.x;
  if (a.prof && tid == 0) {
    const unsigned long long t0 = fused_now();
    if (blockIdx.x == 0) a.prof[0] = t0;
    if (a.spec) {
      fused_bstamp(a, 0, t0);
      for (uint32_t k = 7; k < kProfBlockWords; ++k) fused_bstamp(a, k, 0);
    }
  }
  if (tid == 0) {
    const FusedScalars sc = a.sc_dev ? *a.sc_dev : a.sc;
    s_dyn = sc.dyn;
    s_seq = sc.seq;
    s_kept_fp = sc.kept_fp;
    s_zc_in = reinterpret_cast<unsigned long long>(sc.zc_in);
    s_zc_out = reinterpret_cast<unsigned long long>(sc.zc_out);
    if (blockIdx.x == 0 && a.dyn_out) *a.dyn_out = sc.dyn;
  }
  __syncthreads();
  const uint32_t n = s_dyn.n;
  const uint32_t nb_live = (n + 1023) / 1024;            // request tiles that hold requests
  const uint32_t m = (uint32_t)*a.m_ptr;
  const uint32_t lt_live = min((m + kListTile - 1) / kListTile, a.n_ltiles);  // slot tiles that hold slots
  const ReqView rv{a.reqs, a.reqs16};

  if (tid < 64) s_seen[tid] = kClsEmpty;
  __syncthreads();
  {
    const size_t S4 = size_t(a.n_servants) * 4;
    if (a.spec) {
      fused_prefetch(a.kept_env, size_t(a.t.n_envs) * sizeof(uint4));
      fused_prefetch(a.t.ip_comp_mask, size_t(a.t.n_ips) * 8);
      // (fused_servant_counters)
      fused_prefetch(a.kept_sv, S4);
      fused_prefetch(a.sv.ever, S4 * 2);
      fused_prefetch(a.dec.row_off, S4);
      fused_prefetch(a.dec.row_len, S4);
      fused_prefetch(a.slot_spos, size_t(m) * 4);
    }
    fused_prefetch(a.dec.rec, size_t(m) * 8);
    fused_prefetch(a.sv.run, S4);
    fused_prefetch(a.sv.version, S4);
    fused_prefetch(a.sv.max_tasks, S4);
    fused_prefetch(a.t.sv_comp, S4);
    fused_prefetch(a.t.sv_local, S4);
    fused_prefetch(a.t.comp_sv, S4);
    if (a.t.sv_emask) fused_prefetch(a.t.sv_emask, S4 * 2);
    else { fused_prefetch(a.t.sv_env_off, S4 + 4); }
  }
  const char* zc_in = reinterpret_cast<const char*>(s_zc_in);
  uint32_t ncls, nlists;
  const bool lite = a.solo && a.loff_cache_words != 0;  // (the host speculates only when it holds)
  // speculative: class | in-tile rank << 16 of this thread's request in the block's first / second request tile
  uint32_t spec_cr0 = 0xffffu, spec_cr1 = 0xffffu;
  if (a.spec) {
    // ---- A: requests against the kept class table, list ballots and counts, eligible servants per class ------------
    // Request tiles are the first items, so tile t is handled by block t % G here and in B below: the class and rank of
    // a request stay in this thread's registers.
    __shared__ uint32_t s_cls_mv[kMaxClasses];
    ncls = min(a.ct.meta[0], a.ct.cls_bound);
    nlists = min(a.ct.meta[3], a.ct.cls_bound);
    bool miss = false, facts = false;
    const uint32_t items = nb_live + lt_live + ncls;
    uint32_t kinds = 0;  // (YDSCHED_FUSED_PROF)
    for (uint32_t it = blockIdx.x, k = 0; it < items; it += G, ++k) {
      uint32_t kind;
      if (it < nb_live) {
        uint32_t env, mv, ip, cls = kNone;
        if (fused_fetch_req(a, rv, zc_in, it, n, env, mv, ip)) cls = kept_class(env, mv, ip, a.t, a.kept_env, miss);
        const uint32_t rank = rank_in_tile(it, cls, a.ct, a.n_rtiles, a.rank_cnt);
        const uint32_t cr = (rank << 16) | (cls & 0xffffu);
        if (k == 0) spec_cr0 = cr;
        else if (k == 1) spec_cr1 = cr;
        else miss = true;  // (more request tiles than two per block: the host does not speculate on such batches)
        kind = kItemRequests;
      } else if (it < nb_live + lt_live) {
        list_count_tile_kept(it - nb_live, m, ncls, a.dec, a.ct, a.sv, a.kept_sv, a.n_ltiles, a.list_cnt, a.members,
                             s_cls_mv, facts);
        kind = kItemSlots;
      } else {
        cls_elig_class(it - nb_live - lt_live, a.t, a.ct, a.sv);
        kind = kItemClass;
      }
      if (a.prof && k < kProfMaxItems) {
        __syncthreads();  // (the item's end: all of its threads are done)
        fused_bstamp(a, 1 + k, fused_now());
        kinds |= kind << (4 * k);
      }
      if (a.prof) fused_bstamp(a, 7, kinds | (min(k + 1, 0xffffu) << 16));
    }
    // slot tiles beyond the table's end hold no members (the lists' row scans below read them; nothing re-zeroes them)
    const uint32_t tail = a.n_ltiles - lt_live;
    for (uint32_t i = blockIdx.x * 1024 + tid; i < nlists * tail; i += G * 1024) a.list_cnt[(i / tail) * a.n_ltiles + lt_live + i % tail] = 0;
    // (meta[1] is for the report; the barrier tells the blocks)
    if (__any_sync(0xffffffffu, miss) && (tid & 31) == 0) atomicExch(&a.ct.meta[1], kFlagSpecMiss);
    fused_stamp(a, 1);
    fused_bstamp(a, 4, fused_now());
    const bool missed = fused_barrier_any(a.bar, 1, miss);
    fused_stamp(a, 2);
    fused_bstamp(a, 5, fused_now());
    if (missed) {
      // nothing is decided: the last block reports and leaves the scratch clean (the kept table too) for the replay
      if (fused_done_last(a.bar)) {
        fused_report(a, s_seq, 0);
        __syncthreads();  // (the report reads meta[], which lies in the region zeroed below)
        for (uint32_t i = tid; i < kClsTableSize; i += 1024) a.clean_keys[i] = kClsEmpty;
        for (uint32_t i = tid; i < a.clean_zero_vec; i += 1024) a.clean_zero[i] = make_uint4(0u, 0u, 0u, 0u);
      }
      return;
    }
  } else {
  // ---- P1: classes ---------------------------------------------------------------------------------------------
  for (uint32_t tile = blockIdx.x; tile < nb_live; tile += G) {
    uint32_t env, mv, ip;
    if (fused_fetch_req(a, rv, zc_in, tile, n, env, mv, ip)) cls_insert_one(env, mv, ip, a.t, a.ct, s_seen);
  }

  fused_stamp(a, 1);
  // ---- E1: class numbering and solver modes, by the last block to arrive ------------------------------------------
  if (fused_arrive(a.bar, 1)) {
    cls_finalize_block(a.t, a.ct, a.n_comps, a.comp_mode, a.solo);
    fused_release(a.bar, 1);
  } else {
    fused_wait(a.bar, 1);
  }
  // Overflow (1, 2) or a solo kernel facing a coupled component (4): nothing is decided, the host replays the batch.
  // Every block reads the same value: nobody writes the flag between E1's release and the next barrier's arrival
  // ... except list_fill_tile (P5), which is behind E2; the check is repeated after B3.
  if (*reinterpret_cast<volatile uint32_t*>(&a.ct.meta[1]) != 0) {
    if (a.solo && blockIdx.x == 0) fused_report(a, s_seq, 0);
    return;
  }
  ncls = min(a.ct.meta[0], a.ct.cls_bound);
  nlists = min(a.ct.meta[3], a.ct.cls_bound);
  fused_stamp(a, 2);

  // ---- P3: rank counts, list ballots and counts, eligible servants per class ---------------------------------------
  {
    const uint32_t items = lt_live + a.n_rtiles + ncls;
    for (uint32_t it = blockIdx.x; it < items; it += G) {
      if (it < lt_live) {
        list_count_tile(it, m, a.dec, a.t, a.ct, a.sv, a.n_ltiles, a.list_cnt, a.list_bal, a.solo ? a.members : nullptr);
      } else if (it < lt_live + a.n_rtiles) {
        const uint32_t tile = it - lt_live;
        if (tile < nb_live) {
          rank_count_tile(tile, rv, n, a.t, a.ct, a.comp_mode, a.n_rtiles, a.rcls, a.rrank, a.rself, a.rank_cnt);
        } else if (tid < a.ct.cls_bound) {  // beyond the queue's end: empty cells (the matrix is not pre-zeroed)
          a.rank_cnt[tid * a.n_rtiles + tile] = 0;
        }
      } else {
        cls_elig_class(it - lt_live - a.n_rtiles, a.t, a.ct, a.sv);
      }
    }
  }

  fused_stamp(a, 3);
  // ---- E2: both count matrices -> offsets (class-major, tile-minor, + the end cell) -------------------------------
  if (lite) {
    fused_barrier(a.bar, 2);  // the counts stay raw: each block derives what it needs below
  } else if (fused_arrive(a.bar, 2)) {
    fused_scan_flat(a.rank_cnt, ncls * a.n_rtiles + 1);
    fused_scan_flat(a.list_cnt, nlists * a.n_ltiles + 1);
    fused_release(a.bar, 2);
  } else {
    fused_wait(a.bar, 2);
  }
  }

  fused_stamp(a, 4);
  if (!a.solo) {
  // ---- P5: per-class sorted slot lists (the coupled solvers read them) -------------------------------------------
  for (uint32_t tile = blockIdx.x; tile < lt_live; tile += G) {
    list_fill_tile(tile, m, a.dec, a.t, a.ct, a.n_ltiles, a.list_cnt, a.list_bal, a.list, a.list_cap);
  }

  fused_stamp(a, 5);
  // ---- B3 ---------------------------------------------------------------------------------------------------------
  if (fused_arrive(a.bar, 3)) fused_release(a.bar, 3);
  else fused_wait(a.bar, 3);
  if (*reinterpret_cast<volatile uint32_t*>(&a.ct.meta[1]) != 0) return;  // a list outgrew its buffer: nothing is decided
  }

  fused_stamp(a, 6);
  // ---- P6: verdicts (+ solo: ids, grants, leases) -----------------------------------------------------------------
  const long long now_ns = s_dyn.now_ns;
  TaskRing ring = a.ring;
  ring.next = s_dyn.ring_next;
  void* const out = s_zc_out ? reinterpret_cast<void*>(s_zc_out) : a.out;
  if (lite) {
    // every component with requests is data-parallel: no lists, each request's member is picked from the per-tile member
    // lists; the tables the selection searches are built here, per block, from the raw (class, tile) counts.  Every load
    // of those tables, the request's class and rank (not speculative) and its lease fields (final_tile) are issued before
    // the first wait: one round trip to L2, then shared memory, then the member load.
    __shared__ uint32_t s_rpre[kMaxClasses];   // class-c requests in the request tiles before this one
    __shared__ uint32_t s_nelig[kMaxClasses];  // cls_nelig
    __shared__ uint32_t s_base;                // grants of the request tiles before this one
    const uint32_t lane = tid & 31, warp = tid >> 5, stride = a.n_ltiles + 1, cells = nlists * a.n_ltiles;
    for (uint32_t tile = blockIdx.x, k = 0; tile < nb_live; tile += G, ++k) {
      const uint32_t q = tile * 1024 + tid;
      uint32_t c = kNone, rank = 0, lflags = 0;  // rank: among the class's requests of this tile
      long long lexp = 0;
      if (q < n) {
        rv.lease(q, lflags, lexp);
        if (a.spec) {
          const uint32_t cr = k == 0 ? spec_cr0 : spec_cr1;
          if ((cr & 0xffffu) != 0xffffu) { c = cr & 0xffffu; rank = cr >> 16; }
        } else {
          c = a.rcls[q];
          rank = a.rrank[q];
        }
      }
      uint32_t cnt0 = 0, nelig = 0;  // (first tile) this thread's first (class, slot tile) count, class tid's cls_nelig
      if (k == 0) {
        if (tid < cells) cnt0 = a.list_cnt[tid];
        if (tid < ncls) nelig = a.ct.cls_nelig[tid];
      }
      if (tid == 0) s_base = 0;
      for (uint32_t cc = warp; cc < ncls; cc += 32) {  // class-cc requests in the tiles before this one
        uint32_t sum = 0;
        for (uint32_t t0 = 0; t0 < tile; t0 += 4 * 32) {
          uint32_t v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint32_t t = t0 + u * 32 + lane;
            v[u] = t < tile ? a.rank_cnt[cc * a.n_rtiles + t] : 0u;
          }
          sum += v[0] + v[1] + v[2] + v[3];
        }
        sum = __reduce_add_sync(0xffffffffu, sum);
        if (lane == 0) s_rpre[cc] = sum;
      }
      if (k == 0) {
        if (tid < cells) s_loff[(tid / a.n_ltiles) * stride + tid % a.n_ltiles] = cnt0;
        for (uint32_t i = tid + 1024; i < cells; i += 1024) s_loff[(i / a.n_ltiles) * stride + i % a.n_ltiles] = a.list_cnt[i];
        if (tid < ncls) s_nelig[tid] = nelig;
      }
      __syncthreads();
      // (first tile) class cc's row of counts -> row-local exclusive offsets of its slot tiles + its total, in place;
      // then the class's grants in the request tiles before this one
      for (uint32_t cc = warp; cc < nlists; cc += 32) {
        uint32_t* row = s_loff + cc * stride;
        uint32_t running = 0;
        if (k == 0) {
          for (uint32_t t0 = 0; t0 < a.n_ltiles; t0 += 32) {
            const uint32_t t = t0 + lane;
            const uint32_t v = t < a.n_ltiles ? row[t] : 0u;
            uint32_t x = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
              const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
              if (lane >= d) x += y;
            }
            if (t < a.n_ltiles) row[t] = running + x - v;
            running += __shfl_sync(0xffffffffu, x, 31);
          }
          if (lane == 0) row[a.n_ltiles] = running;
        } else {
          running = row[a.n_ltiles];
        }
        if (lane == 0 && cc < ncls) {
          const uint32_t g = fused_class_grants(s_nelig[cc], s_rpre[cc], running);
          if (g) atomicAdd(&s_base, g);
        }
      }
      __syncthreads();
      const uint32_t base = s_base;
      const bool stamp = a.prof && a.spec && k == 0;
      if (stamp) fused_bstamp(a, 8, fused_now());
      const uint32_t r = c != kNone ? fused_select(c, s_rpre[c] + rank, a, s_nelig, s_loff, stride) : kResEnvNotFound;
      if (stamp) {
        __syncthreads();  // (every selection of the tile is done)
        fused_bstamp(a, 9, fused_now());
      }
      if (a.spec) {  // (the servant counters are counted below)
        if (a.packed_out) final_tile<true, true, true, true, false>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base, lflags, lexp);
        else final_tile<false, true, true, true, false>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base, lflags, lexp);
      } else {
        if (a.packed_out) final_tile<true, true, true, true>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base, lflags, lexp);
        else final_tile<false, true, true, true>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base, lflags, lexp);
      }
      if (stamp) fused_bstamp(a, 10, fused_now());  // (final_tile ends with a block barrier)
    }
    if (a.spec) {
      const bool idle = G >= nb_live + kCounterMinBlocks;  // enough blocks without a request tile
      if (!idle || blockIdx.x >= nb_live) {
        fused_servant_counters(a, ncls, nb_live, idle ? blockIdx.x - nb_live : blockIdx.x, idle ? G - nb_live : G);
        if (a.prof) {
          __syncthreads();
          fused_bstamp(a, 11, fused_now());
        }
      }
    }
  } else if (a.solo) {
    // (offsets too big for shared memory: scanned by the leader of E2)
    const uint32_t* loff = a.list_cnt;
    for (uint32_t tile = blockIdx.x; tile < nb_live; tile += G) {
      uint32_t before = 0;  // (thread c) grants of class c in the tiles before this one, from the scanned counts
      if (tid < ncls) {
        const uint32_t* rrow = a.rank_cnt + tid * a.n_rtiles;
        before = fused_class_grants(a.ct.cls_nelig[tid], rrow[tile] - rrow[0], loff[(tid + 1) * a.n_ltiles] - loff[tid * a.n_ltiles]);
      }
      const uint32_t base = fused_block_sum(before);
      const uint32_t q = tile * 1024 + tid;
      uint32_t r = kResEnvNotFound;
      const uint32_t c = q < n ? a.rcls[q] : kNone;  // (kNone: an unknown digest, or one nobody holds)
      if (c != kNone) {
        const uint32_t* rrow = a.rank_cnt + c * a.n_rtiles;
        r = fused_select(c, rrow[q / kRankTile] - rrow[0] + a.rrank[q], a, a.ct.cls_nelig, loff, a.n_ltiles);
      }
      if (a.packed_out) final_tile<true, true, true>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base);
      else final_tile<false, true, true>(tile, nb_live - 1, r, n, now_ns, rv, nullptr, a.comp_sv, ring, out, a.counters, a.sv.run, a.sv.ever, base);
    }
  } else {
    for (uint32_t tile = blockIdx.x; tile < nb_live; tile += G) {
      const uint32_t q = tile * 1024 + tid;
      uint32_t v;
      if (q < n && rank_assign_one(q, a.n_rtiles, a.t, a.ct, a.rcls, a.rrank, a.rself, a.rank_cnt, a.list_cnt, a.n_ltiles,
                                   a.list, a.comp_mode, a.rq, a.L, v)) {
        a.res[q] = v;
      }
    }
  }
  fused_stamp(a, 7);
  if (a.spec && a.prof) {
    __syncthreads();  // (every thread of the block is done with B)
    fused_bstamp(a, 6, fused_now());
  }
  // ---- solo: the block that finishes last reports to the host and leaves the scratch as the next solve expects it ----
  // A speculative solve resets the barrier words alone: the class table stays, and everything else it wrote is
  // rewritten by the next one before it is read.  Any other solo solve keeps its class table when its class set is the
  // one of the previous solve (the host speculates next), else it clears the table; the rest of the scratch is zeroed.
  if (a.solo && fused_done_last(a.bar)) {
    if (a.spec) {
      fused_report(a, s_seq, a.counters->granted);
      if (tid < 3) a.bar[tid] = 0;
    } else {
      const unsigned long long fp = fused_classes_fp(a.clean_keys);
      fused_report(a, s_seq, a.counters->granted, fp);
      __syncthreads();  // (the report reads meta[], which lies in the region zeroed below)
      uint32_t from = 0;
      if (fp == s_kept_fp) {
        from = kKeptClsWords / 4;
        fused_keep_env(a);
      } else {
        for (uint32_t i = tid; i < kClsTableSize; i += 1024) a.clean_keys[i] = kClsEmpty;
      }
      for (uint32_t i = from + tid; i < a.clean_zero_vec; i += 1024) a.clean_zero[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (a.prof && tid == 0) a.prof[8] = fused_now();
  }
}

// Converts a packed upload into the 24-byte queue (the sequences that do not start with k_fused_front).
__global__ void __launch_bounds__(256) k_unpack_reqs(const uint4* __restrict__ reqs16, const DynParams* __restrict__ dp,
                                                     yd_task_req* __restrict__ reqs) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= dp->n) return;
  const uint4 w = __ldg(reqs16 + q);
  uint2* dst = reinterpret_cast<uint2*>(reqs + q);
  const unsigned long long ns = (unsigned long long)(w.w & 0x7fffffffu) * 1000000ull;
  dst[0] = make_uint2(w.x, w.y);
  dst[1] = make_uint2(w.z, (w.w >> 31) ? YD_REQ_FLAG_PREFETCH : 0u);
  dst[2] = make_uint2((uint32_t)ns, (uint32_t)(ns >> 32));
}

// 16-byte grants -> 8-byte grants (the sequences that do not end inside k_fused_front).  task_id - first_id is the
// grant's FIFO ordinal when ids are dense; with strided ids (sharded deployments) it is (task_id - first) / stride.
__global__ void __launch_bounds__(256) k_pack_grants(const uint4* __restrict__ grants, const DynParams* __restrict__ dp,
                                                     TaskRing ring, uint2* __restrict__ out) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= dp->n) return;
  const uint4 g = grants[q];  // {id lo, id hi, servant, status}
  uint32_t ordinal = 0;
  if (g.w == YD_STATUS_GRANTED) {
    const unsigned long long xid = ((unsigned long long)g.y << 32) | g.x;
    unsigned long long local = 0;
    ring.loc(xid, &local);
    ordinal = (uint32_t)(local - dp->ring_next);
  }
  out[q] = make_uint2(g.z, (g.w << 30) | ordinal);
}

}  // namespace yd
