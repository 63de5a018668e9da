// classes.cuh -- request classes and their sorted slot lists (slot-stream solver).
//
// A *class* is what UnsafeEnumerateEligibleServants keys on: (compiler digest,
// min_version) (task_dispatcher.cc:316-344).  All requests of a class see the same
// eligible servants, hence the same candidate slots in the same order; the only
// per-request difference is which servant is "self" (cc:372-379).
//
//   k_cls_insert   every request inserts its (digest id, min_version) into a small
//                  open-addressing table in HBM (atomicCAS on 8-byte keys) and flags
//                  its component if the requestor's IP matches a servant there
//   k_cls_number   one block numbers the occupied table slots in slot order
//                  (deterministic ids) and records digest / min_version / component
//   k_cls_elig     per class: number of eligible servants (0 => EnvironmentNotFound)
//   k_slot_decode  sorted slot -> (registry position, running_tasks value, component)
//   k_list_count / k_list_fill   per class, order-preserving filter of the sorted
//                  slots by class eligibility -> L[c] = (servant local index, r)
#pragma once
#include "common.cuh"

namespace yd {

constexpr uint32_t kClsTableSize = 2048;  // power of two
constexpr uint32_t kMaxClasses = 256;
constexpr unsigned long long kClsEmpty = ~0ull;

struct ClassTable {
  unsigned long long* keys;  // [kClsTableSize] digest id << 32 | min_version, or kClsEmpty
  uint32_t* slot_cls;        // [kClsTableSize] class id of the slot
  uint32_t* meta;            // [0] number of classes, [2] number of merge-mode components, [1] overflow flag (1: too many classes / table full / list
                             //     too long -> row-scan solver; 2: more classes than cls_bound -> retry with a bigger bound)
  uint32_t cls_bound;        // classes the per-class grids / tables of this solve are sized for (<= kMaxClasses)
  uint32_t* cls_env;         // [kMaxClasses]
  uint32_t* cls_mv;
  uint32_t* cls_comp;
  uint32_t* cls_nelig;       // eligible servants (max_tasks != 0, digest, version)
  uint32_t* cls_count;       // requests of the class in this batch
  uint32_t* cls_lbit;        // index of the class among the classes of its component (merge solver)
  uint32_t* comp_flags;      // [C] bit 0: some requestor's IP is that of exactly ONE servant of the component ("self",
                             //     cc:372-379); bit 1: of several servants of the component (self = the first FREE one)
  uint32_t* comp_ncls;       // [C] classes in the component
  uint32_t* comp_midx;       // [C] merge-mode components: index of their pseudo-class list, else kNone
  uint32_t* merge_comp;      // [cls_bound] pseudo-class index -> component
  uint32_t* comp_cls;        // [cls_bound * 32] (pseudo-class index, class index inside the component) -> class id
  uint32_t force_stream;     // 1 (test switch): components with self-requests go to the sequential solver;
                             // 2: so does everything the merge solver would take (its last-ditch retry)
};

struct TopoView {  // the parts of the topology the class kernels need
  const uint32_t* env_comp;
  uint32_t n_envs;
  const uint32_t* sv_comp;
  const uint32_t* sv_local;
  const uint32_t* ip_off;
  const uint32_t* ip_sv;
  uint32_t n_ips;
  const uint32_t* sv_env_off;  // CSR: registry position -> digest ids it holds
  const uint32_t* sv_envs;
  const uint32_t* comp_sv_off;
  const uint32_t* comp_sv;
  // digest membership as one 64-bit word per servant (bit = the digest's index inside its component, env_local), or
  // null when some component holds more than 64 digests (the CSR above is walked instead)
  const unsigned long long* sv_emask;
  const uint32_t* env_local;
  // per requestor IP (< n_ips): bit c = some servant of component c (< 64) is on that IP (ip_off / ip_sv in one load)
  const unsigned long long* ip_comp_mask;
};

__device__ __forceinline__ uint32_t cls_hash(unsigned long long key) {
  key ^= key >> 33;
  key *= 0xff51afd7ed558ccdULL;
  key ^= key >> 29;
  return (uint32_t)key & (kClsTableSize - 1);
}

// Returns the table slot holding `key`, or kNone if absent (lookup only).
__device__ __forceinline__ uint32_t cls_find(const unsigned long long* __restrict__ keys, unsigned long long key) {
  uint32_t s = cls_hash(key);
  for (uint32_t probe = 0; probe < kClsTableSize; ++probe) {
    unsigned long long k = keys[s];
    if (k == key) return s;
    if (k == kClsEmpty) return kNone;
    s = (s + 1) & (kClsTableSize - 1);
  }
  return kNone;
}

__device__ __forceinline__ bool servant_has_env(const TopoView& t, uint32_t pos, uint32_t env) {
  if (t.sv_emask) return (t.sv_emask[pos] >> (t.env_local[env] & 63u)) & 1ull;
  for (uint32_t u = t.sv_env_off[pos], e = t.sv_env_off[pos + 1]; u < e; ++u) {
    if (t.sv_envs[u] == env) return true;
  }
  return false;
}

// One request's contribution: its (digest id, min_version) goes into the class table (deduplicated per block through
// the 64-entry shared-memory set `s_seen`, which the caller initialises to kClsEmpty), and its component learns whether
// the requestor's IP belongs to one / several of its servants.
__device__ __forceinline__ void cls_insert_one(uint32_t env, uint32_t mv, uint32_t ip, const TopoView& t,
                                               const ClassTable& ct, unsigned long long* s_seen) {
  if (env >= t.n_envs) return;
  const uint32_t comp = t.env_comp[env];
  if (comp == kNone) return;
  const unsigned long long key = ((unsigned long long)env << 32) | mv;
  // A batch has few classes and 100 k requests: dedupe inside the block first (a 64-slot
  // shared-memory set), so the HBM table sees ~one insert per (block, class).
  bool first_in_block = true;
  {
    uint32_t h = cls_hash(key) & 63u;
    for (int probe = 0; probe < 64; ++probe) {
      unsigned long long k = s_seen[h];
      if (k == kClsEmpty) k = atomicCAS(&s_seen[h], kClsEmpty, key);
      if (k == key) { first_in_block = false; break; }   // somebody in this block has it
      if (k == kClsEmpty) break;                         // I claimed the slot: I insert globally
      h = (h + 1) & 63u;
    }
  }
  if (first_in_block) {
    uint32_t s = cls_hash(key);
    bool done = false;
    for (uint32_t probe = 0; probe < kClsTableSize && !done; ++probe) {
      unsigned long long k = ct.keys[s];
      if (k == kClsEmpty) k = atomicCAS(&ct.keys[s], kClsEmpty, key);
      if (k == key || k == kClsEmpty) done = true;
      else s = (s + 1) & (kClsTableSize - 1);
    }
    if (!done) atomicExch(&ct.meta[1], 1u);  // table full -> caller falls back to the row-scan solver
  }
  // does the requestor's IP belong to one / several servants of this component?
  if (ip < t.n_ips) {
    uint32_t mine = 0;
    for (uint32_t u = t.ip_off[ip], e = t.ip_off[ip + 1]; u < e && mine < 2; ++u) {
      if (t.sv_comp[t.ip_sv[u]] == comp) ++mine;
    }
    const uint32_t bit = mine >= 2 ? 2u : mine;
    if (bit && !(ct.comp_flags[comp] & bit)) atomicOr(&ct.comp_flags[comp], bit);
  }
}

// The kept class table as seen from a digest (fused.cuh, speculative variant): kept_env[env] = {class, its min_version,
// its component, 0}, where the class is the one the digest's component holds in the table -- a kept table holds at most
// one class per component, and only if that class is of this digest -- or x = kNone (no component holds the digest) or
// x = kKeptNoClass (its component holds no class of this digest).
constexpr uint32_t kKeptNoClass = 0xFFFFFFFEu;

// A request's class in the table a previous solo solve kept, or kNone for an unknown digest or one no component holds
// (EnvironmentNotFound, as cls_insert_one skips them).  `miss`: the kept table cannot decide the request -- its class is
// not in the table, or the requestor's IP is that of a servant of the component (which would take it off the
// data-parallel path).  Two independent loads after the request: the digest's kept_env word and the IP's component mask
// (the IP CSR is walked only for a component beyond the mask's 64 bits).
__device__ __forceinline__ uint32_t kept_class(uint32_t env, uint32_t mv, uint32_t ip, const TopoView& t,
                                               const uint4* __restrict__ kept_env, bool& miss) {
  if (env >= t.n_envs) return kNone;
  const uint4 w = kept_env[env];
  const unsigned long long ipm = ip < t.n_ips ? t.ip_comp_mask[ip] : 0ull;
  if (w.x == kNone) return kNone;
  if (w.x == kKeptNoClass || w.y != mv) {
    miss = true;
    return kNone;
  }
  const uint32_t comp = w.z;
  if (comp < 64) {
    if ((ipm >> comp) & 1ull) miss = true;
  } else if (ip < t.n_ips) {
    for (uint32_t u = t.ip_off[ip], e = t.ip_off[ip + 1]; u < e; ++u) {
      if (t.sv_comp[t.ip_sv[u]] == comp) miss = true;
    }
  }
  return w.x;
}

__global__ void __launch_bounds__(256) k_cls_insert(const yd_task_req* __restrict__ reqs,
                                                    const DynParams* __restrict__ dp, TopoView t, ClassTable ct) {
  __shared__ unsigned long long s_seen[64];
  if (threadIdx.x < 64) s_seen[threadIdx.x] = kClsEmpty;
  __syncthreads();
  uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= dp->n) return;
  const uint2 w0 = __ldg(reinterpret_cast<const uint2*>(reqs + q));
  const uint32_t ip = __ldg(reinterpret_cast<const uint2*>(reqs + q) + 1).x;
  cls_insert_one(w0.x, w0.y, ip, t, ct, s_seen);
}

// The requestor's own servant as the solvers see it: component-local index of the ONE servant of
// component `comp` whose observed location is on the requestor's IP (IsNetworkAddressEqual,
// cc:66-69), else kNone.  (Several such servants: the component takes the sequential solver.)
__device__ __forceinline__ uint32_t self_servant(const TopoView& t, uint32_t ip, uint32_t comp) {
  uint32_t self = kNone, mine = 0;
  if (ip < t.n_ips) {
    for (uint32_t u = t.ip_off[ip], e = t.ip_off[ip + 1]; u < e; ++u) {
      const uint32_t p = t.ip_sv[u];
      if (t.sv_comp[p] == comp) { self = t.sv_local[p]; ++mine; }
    }
  }
  return mine == 1 ? self : kNone;
}

// Range-sharded queue: every rank has inserted the classes of ITS requests; `gathered` holds all the
// ranks' tables (per rank `stride` u32 words: kClsTableSize 8-byte keys, then n_comps component flags).
// One warp rebuilds the table from them in a fixed order (rank-major, slot order, one insert at a
// time), so every rank ends up with the SAME table -- and therefore the same class ids, lists and
// solver modes -- and ORs the flags.
__global__ void __launch_bounds__(32) k_cls_merge_tables(const uint32_t* __restrict__ gathered, uint32_t stride,
                                                         uint32_t world, uint32_t n_comps, ClassTable ct) {
  const uint32_t lane = threadIdx.x;
  for (uint32_t i = lane; i < kClsTableSize; i += 32) ct.keys[i] = kClsEmpty;
  for (uint32_t c = lane; c < n_comps; c += 32) {
    uint32_t f = 0;
    for (uint32_t g = 0; g < world; ++g) f |= gathered[size_t(g) * stride + 2 * kClsTableSize + c];
    ct.comp_flags[c] = f;
  }
  __syncwarp();
  for (uint32_t g = 0; g < world; ++g) {
    const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(gathered + size_t(g) * stride);
    for (uint32_t s0 = 0; s0 < kClsTableSize; s0 += 32) {
      const unsigned long long key = keys[s0 + lane];
      uint32_t todo = __ballot_sync(0xffffffffu, key != kClsEmpty);
      while (todo) {
        const uint32_t b = __ffs(todo) - 1;
        todo &= todo - 1;
        if (lane == b) {
          uint32_t s = cls_hash(key);
          bool done = false;
          for (uint32_t probe = 0; probe < kClsTableSize && !done; ++probe) {
            const unsigned long long k = ct.keys[s];
            if (k == kClsEmpty) { ct.keys[s] = key; done = true; }
            else if (k == key) done = true;
            else s = (s + 1) & (kClsTableSize - 1);
          }
          if (!done) ct.meta[1] = 1;
        }
        __syncwarp();
      }
    }
  }
}

// One block: deterministic class ids (= rank of the occupied table slot), per-class
// eligible-servant counts, and the solver mode of every component:
//   comp_mode 1 = data-parallel path (one class, no request from one of its own servants),
//             0 = sequential slot-stream solver.
// (A block of 1024 threads.  `solo`: the caller can only finish batches made of data-parallel components by itself
// (fused.cuh); anything else raises flag 4 = "run the general sequence".  meta[4] tells the host either way.)
__device__ __forceinline__ void cls_finalize_block(const TopoView& t, const ClassTable& ct, uint32_t n_comps,
                                                   uint32_t* __restrict__ comp_mode, uint32_t solo) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  __shared__ uint32_t s_other;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry_s = 0; s_other = 0; }
  __syncthreads();
  for (uint32_t base = 0; base < kClsTableSize; base += 1024) {
    const uint32_t s = base + tid;
    const unsigned long long k = ct.keys[s];
    const uint32_t v = k != kClsEmpty ? 1u : 0u;
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
    const uint32_t id = carry_s + (warp ? warp_sums[warp - 1] : 0) + x - v;
    if (v) {
      if (id < kMaxClasses) {
        ct.slot_cls[s] = id;
        const uint32_t env = (uint32_t)(k >> 32);
        const uint32_t comp = t.env_comp[env];
        ct.cls_env[id] = env;
        ct.cls_mv[id] = (uint32_t)k;
        ct.cls_comp[id] = comp;
        atomicAdd(&ct.comp_ncls[comp], 1u);
      } else {
        ct.slot_cls[s] = kNone;
        ct.meta[1] = 1;
      }
      if (id >= ct.cls_bound && id < kMaxClasses) atomicMax(&ct.meta[1], 2u);  // 1 (hard overflow) wins below
    }
    __syncthreads();
    if (tid == 1023) carry_s += warp_sums[31];
    __syncthreads();
  }
  const uint32_t ncls = carry_s < kMaxClasses ? carry_s : kMaxClasses;
  if (tid == 0) {
    ct.meta[0] = ncls;
    if (carry_s > kMaxClasses) ct.meta[1] = 1;
  }
  __threadfence_block();
  __syncthreads();
  // index of each class among the classes of its component
  for (uint32_t c = tid; c < ncls; c += 1024) {
    uint32_t lb = 0;
    const uint32_t comp = ct.cls_comp[c];
    for (uint32_t o = 0; o < c; ++o) lb += ct.cls_comp[o] == comp ? 1u : 0u;
    ct.cls_lbit[c] = lb;
  }
  // solver mode per component:
  //   1 = data-parallel (one class, nobody requests from one of its own servants)
  //   2 = merge solver  (1..32 classes; requestors may be servants of the component, but no IP
  //       carries several of its servants)
  //   0 = sequential slot-stream solver
  const bool healthy = ct.meta[1] == 0;
  __shared__ uint32_t s_nmerge;
  if (tid == 0) s_nmerge = 0;
  __syncthreads();
  for (uint32_t c = tid; c < n_comps; c += 1024) {
    uint32_t mode = 0, midx = kNone;
    const uint32_t k = ct.comp_ncls[c];
    const uint32_t fl = ct.comp_flags[c];
    if (healthy && !(fl & 2u) && !(ct.force_stream == 1 && (fl & 1u))) {
      if (k == 1 && !(fl & 1u)) mode = 1;
      else if (ct.force_stream != 2 && k >= 1 && k <= 32) {
        midx = atomicAdd(&s_nmerge, 1u);
        if (ncls + midx < ct.cls_bound) { mode = 2; ct.merge_comp[midx] = c; }
        else { midx = kNone; atomicMax(&ct.meta[1], 2u); }  // needs a bigger per-class grid: retry
      }
    }
    comp_mode[c] = mode;
    ct.comp_midx[c] = midx;
    if (k >= 1 && mode != 1) s_other = 1;  // requests for a component the data-parallel path cannot decide
  }
  __syncthreads();
  for (uint32_t c = tid; c < ncls; c += 1024) {
    const uint32_t midx = ct.comp_midx[ct.cls_comp[c]];
    if (midx != kNone && ct.cls_lbit[c] < 32) ct.comp_cls[midx * 32 + ct.cls_lbit[c]] = c;
  }
  if (tid == 0) {
    ct.meta[2] = s_nmerge;
    ct.meta[3] = min(ncls + s_nmerge, ct.cls_bound);  // lists to build: classes + merge pseudo-classes
    ct.meta[4] = s_other;
    if (solo && s_other && ct.meta[1] == 0) ct.meta[1] = 4;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(1024) k_cls_finalize(TopoView t, ClassTable ct, ServantArrays sv, uint32_t n_comps,
                                                       uint32_t* __restrict__ comp_mode) {
  cls_finalize_block(t, ct, n_comps, comp_mode, 0u);
}

// Eligible servants per class: max_tasks != 0, digest held, version >= min_version (cc:316-344); 0 => every request
// of the class is EnvironmentNotFound (cc:105-108).  One block per class, beside the list kernels.
__device__ __forceinline__ void cls_elig_class(uint32_t c, const TopoView& t, const ClassTable& ct, const ServantArrays& sv) {
  __shared__ uint32_t s_sum;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  const uint32_t comp = ct.cls_comp[c], env = ct.cls_env[c], mv = ct.cls_mv[c];
  uint32_t mine = 0;
  for (uint32_t i = t.comp_sv_off[comp] + threadIdx.x, e = t.comp_sv_off[comp + 1]; i < e; i += blockDim.x) {
    const uint32_t pos = t.comp_sv[i];
    mine += (sv.max_tasks[pos] != 0 && (uint32_t)sv.version[pos] >= mv && servant_has_env(t, pos, env)) ? 1u : 0u;
  }
  mine = __reduce_add_sync(0xffffffffu, mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_sum, mine);
  __syncthreads();
  if (threadIdx.x == 0) ct.cls_nelig[c] = s_sum;
  __syncthreads();  // (s_sum is reused when a block handles several classes)
}

__global__ void __launch_bounds__(256) k_cls_elig(TopoView t, ClassTable ct, ServantArrays sv) {
  const uint32_t c = blockIdx.x;
  if (c >= min(ct.meta[0], ct.cls_bound)) return;
  cls_elig_class(c, t, ct, sv);
}

// Per-class sorted slot lists.  A block owns a tile of 1024 SORTED slots, decodes each
// slot once (owner position, running_tasks value, component) and loops over the classes:
// class c's list keeps the slots whose servant is eligible for c, in sorted order.
constexpr int kListTile = 1024;

struct SlotDecode {
  const uint32_t* sorted_orig;  // sorted order -> original slot index (radix payload)
  const uint32_t* slot_owner;   // original slot index -> registry position
  const uint32_t* row_off;
  const uint32_t* row_len;
  const uint32_t* run;
  uint32_t static_rows;  // rows hold every running_tasks value from 0 (table kept across solves): slot k of a row IS r = k
  const uint2* rec;      // kept order only (else null): sorted position -> (registry position, r), k_slot_records
};

__device__ __forceinline__ bool decode_slot(const SlotDecode& d, const TopoView& t, uint32_t i, uint32_t m,
                                            uint32_t& pos, uint32_t& r, uint32_t& comp) {
  pos = 0; r = 0; comp = kNone;
  if (i >= m) return false;
  if (d.rec) {  // one load instead of the four dependent ones below
    const uint2 w = d.rec[i];
    if (w.x == kNone) return false;
    pos = w.x; r = w.y;
    if (r < d.run[pos]) return false;  // the servant has filled that slot already
    comp = t.sv_comp[pos];
    return comp != kNone;
  }
  const uint32_t orig = d.sorted_orig[i];
  pos = d.slot_owner[orig];
  const uint32_t k = orig - d.row_off[pos];
  if (k >= d.row_len[pos]) return false;  // (defensive: the stream path's rows carry no sentinel)
  if (d.static_rows) {
    r = k;
    if (r < d.run[pos]) return false;  // the servant has filled that slot already
  } else {
    r = d.run[pos] + k;
  }
  comp = t.sv_comp[pos];
  return comp != kNone;
}

// The kept order's decode, materialised once per rebuild: rec[i] = (registry position, running_tasks value) of sorted
// slot i, or (kNone, 0) for a slot outside its row; and its inverse, spos[row_off[pos] + k] = i, the sorted position of
// every slot of a row (the speculative solve counts a servant's grants from it, fused.cuh: fused_servant_counters).
__global__ void __launch_bounds__(256) k_slot_records(const unsigned long long* __restrict__ m_ptr, SlotDecode d,
                                                      uint2* __restrict__ rec, uint32_t* __restrict__ spos) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint32_t)*m_ptr) return;
  const uint32_t orig = d.sorted_orig[i];
  const uint32_t pos = d.slot_owner[orig];
  const uint32_t k = orig - d.row_off[pos];
  const bool in_row = k < d.row_len[pos];
  rec[i] = in_row ? make_uint2(pos, k) : make_uint2(kNone, 0u);
  if (in_row) spos[orig] = i;
}

// "Slot i belongs to list c" is evaluated ONCE, by the count kernel, as ballots: one 32-bit
// word per (tile, list, warp), kept in HBM (`balg`, row stride cls_bound lists).  The count
// kernel pop-counts them; the fill kernel turns the very same words into in-tile ranks, so the
// two can never disagree about a slot.  Lists are processed in chunks of kListChunk: one or two
// barriers per chunk, whatever the number of classes.
constexpr uint32_t kListChunk = 64;

// The ballots of one chunk of lists, staged for the counts (list_count_tile, list_count_tile_kept: one array per
// kernel, whichever of the two it calls).
__shared__ uint32_t s_count_bal[kListChunk][32];

// Solo solves (fused.cuh) select a list's k-th member straight from per-tile MEMBER LISTS, written where the ballots are
// made: members[(tile * cls_bound + c) * kListTile + j] = the registry position of the j-th member of list c inside slot
// tile `tile` (j = the member's rank in the tile's list: members of the list in lower warps + in lower lanes of its
// warp).  A solo solve's components with requests hold one class each, so a slot is in one list at most.
// The speculative solve's words (list_count_tile_kept) also carry the member's slot index inside the tile above the
// position: pos | slot << kMemberSlotShift.  The host speculates only while the registry holds fewer than 2^22 servants.
__device__ __forceinline__ size_t list_member_index(uint32_t tile, uint32_t c, uint32_t cls_bound) {
  return (size_t(tile) * cls_bound + c) * kListTile;
}
constexpr uint32_t kMemberSlotShift = 22;
constexpr uint32_t kMemberPosMask = (1u << kMemberSlotShift) - 1;
static_assert((1ull << 32 >> kMemberSlotShift) == kListTile, "a member word holds the slot's index inside its tile in its top bits");

// The counts of lists c0 .. c1 in this tile from the chunk's ballots in s_count_bal (warp c - c0 takes list c).
// `prefix`: each ballot word is then replaced by the list's members in the lower warps (the member lists' offsets).
__device__ __forceinline__ void list_chunk_counts(uint32_t c0, uint32_t c1, uint32_t tile, uint32_t n_tiles,
                                                  uint32_t* __restrict__ counts, bool prefix) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t c = c0 + warp; c < c1; c += 32) {
    const uint32_t v = __popc(s_count_bal[c - c0][lane]);
    uint32_t cnt;
    if (prefix) {
      uint32_t x = v;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, s);
        if (lane >= s) x += y;
      }
      s_count_bal[c - c0][lane] = x - v;
      cnt = __shfl_sync(0xffffffffu, x, 31);
    } else {
      cnt = __reduce_add_sync(0xffffffffu, v);
    }
    if (lane == 0) counts[c * n_tiles + tile] = cnt;
  }
}

// `members`: solo solves only (see list_member_index), else null.
__device__ __forceinline__ void list_count_tile(uint32_t tile, uint32_t m, const SlotDecode& d, const TopoView& t,
                                                const ClassTable& ct, const ServantArrays& sv, uint32_t n_tiles,
                                                uint32_t* __restrict__ counts, uint32_t* __restrict__ balg,
                                                uint32_t* __restrict__ members) {
  auto& bal = s_count_bal;
  const uint32_t ncls = min(ct.meta[0], ct.cls_bound);
  const uint32_t nmerge = min(ct.meta[2], ct.cls_bound - ncls);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t pos, r, comp;
  const bool live = decode_slot(d, t, tile * kListTile + tid, m, pos, r, comp);
  const uint32_t ver = live ? (uint32_t)sv.version[pos] : 0u;
  const uint32_t midx = (live && nmerge) ? ct.comp_midx[comp] : kNone;
  uint32_t* my_row = balg + size_t(tile) * ct.cls_bound * 32;
  bool any = false;  // my servant is eligible for some class of its component
  for (uint32_t c0 = 0; c0 < ncls + nmerge; c0 += kListChunk) {
    const uint32_t c1 = min(c0 + kListChunk, ncls + nmerge);
    uint32_t my_c = kNone, my_bal = 0;  // (members) my slot's class list in this chunk, and its ballot
    for (uint32_t c = c0; c < c1; ++c) {
      bool in;
      if (c < ncls) {  // class list: eligibility (cc:316-344)
        in = live && comp == ct.cls_comp[c] && ver >= ct.cls_mv[c] && servant_has_env(t, pos, ct.cls_env[c]);
        any |= in;
      } else {         // pseudo-class of a merge-mode component: every slot some class can use
        in = live && midx == c - ncls && any;
      }
      const uint32_t b = __ballot_sync(0xffffffffu, in);
      if (lane == 0) { bal[c - c0][warp] = b; my_row[c * 32 + warp] = b; }
      if (in && c < ncls) { my_c = c; my_bal = b; }
    }
    __syncthreads();
    list_chunk_counts(c0, c1, tile, n_tiles, counts, members != nullptr);
    if (members) {
      __syncthreads();
      if (my_c != kNone) {
        members[list_member_index(tile, my_c, ct.cls_bound) + bal[my_c - c0][warp] + __popc(my_bal & ((1u << lane) - 1))] = pos;
      }
    }
    __syncthreads();  // the ballots have been consumed
  }
}

// list_count_tile against a kept class table (fused.cuh, speculative variant; ncls classes, no merge pseudo-classes: a
// kept table comes from a solo solve): the same ballot words and counts, with a third of the work.  A slot tile is bound
// by its gathers from random servants and by one eligibility test per (slot, class), not by its load latency; but a kept
// table holds at most one class per component, so a slot is in one list at most -- that of kept_sv[servant] (the class
// of its component, if it holds the class's digest; written with the table), if the servant's version is high enough.
// So: three gathers per slot (run, kept_sv, version) instead of four to five, one test, and the lanes of a warp grouped
// by list (__match_any_sync) instead of one ballot per class.  s_mv: the classes' min_versions in shared memory, loaded
// by the block's first call (`facts`).  It writes the member lists (list_member_index), not the ballot words: the
// speculative solve selects from the member lists alone.  Each word carries the slot's index inside the tile too.
__device__ __forceinline__ void list_count_tile_kept(uint32_t tile, uint32_t m, uint32_t ncls, const SlotDecode& d,
                                                     const ClassTable& ct, const ServantArrays& sv,
                                                     const uint32_t* __restrict__ kept_sv, uint32_t n_tiles,
                                                     uint32_t* __restrict__ counts, uint32_t* __restrict__ members,
                                                     uint32_t* s_mv, bool& facts) {
  auto& bal = s_count_bal;
  uint32_t* const bal_flat = &bal[0][0];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t i = tile * kListTile + tid;
  const uint2 rec = i < m ? d.rec[i] : make_uint2(kNone, 0u);
  const bool load_facts = !facts && tid < ncls;
  const uint32_t f_mv = load_facts ? ct.cls_mv[tid] : 0u;
  const uint32_t pos = rec.x != kNone ? rec.x : 0u;  // (a dead slot reads servant 0's facts: no branch before the loads)
  const uint32_t run = d.run[pos], ver = (uint32_t)sv.version[pos];
  uint32_t cls = kept_sv[pos];
  if (load_facts) s_mv[tid] = f_mv;
  if (!facts) __syncthreads();
  facts = true;
  // a slot outside its row, one the servant has filled already, or a servant below the class's min_version: no list
  if (rec.x == kNone || rec.y < run || cls >= ncls || ver < s_mv[cls]) cls = kNone;
  for (uint32_t c0 = 0; c0 < ncls; c0 += kListChunk) {
    const uint32_t c1 = min(c0 + kListChunk, ncls);
    for (uint32_t k = tid; k < (c1 - c0) * 32; k += kListTile) bal_flat[k] = 0;
    __syncthreads();
    const uint32_t key = (cls >= c0 && cls < c1) ? cls : kNone;
    const uint32_t peers = __match_any_sync(0xffffffffu, key);  // = the ballot of list `key` in this warp
    if (key != kNone && lane == (uint32_t)(__ffs(peers) - 1)) bal[key - c0][warp] = peers;
    __syncthreads();
    list_chunk_counts(c0, c1, tile, n_tiles, counts, true);
    __syncthreads();
    if (key != kNone) {
      members[list_member_index(tile, key, ct.cls_bound) + bal[key - c0][warp] + __popc(peers & ((1u << lane) - 1))] =
          rec.x | tid << kMemberSlotShift;
    }
    __syncthreads();  // the ballots have been consumed
  }
}

__global__ void __launch_bounds__(kListTile) k_list_count(const unsigned long long* __restrict__ m_ptr, SlotDecode d,
                                                          TopoView t, ClassTable ct, ServantArrays sv,
                                                          uint32_t n_tiles, uint32_t* __restrict__ counts,
                                                          uint32_t* __restrict__ balg) {
  list_count_tile(blockIdx.x, (uint32_t)*m_ptr, d, t, ct, sv, n_tiles, counts, balg, nullptr);
}

// counts[] has been exclusive-scanned over (class-major, tile-minor).
__device__ __forceinline__ void list_fill_tile(uint32_t tile, uint32_t m, const SlotDecode& d, const TopoView& t,
                                               const ClassTable& ct, uint32_t n_tiles, const uint32_t* __restrict__ offs,
                                               const uint32_t* __restrict__ balg, uint2* __restrict__ list,
                                               uint32_t list_cap) {
  __shared__ uint32_t bal[kListChunk][32];
  __shared__ uint16_t pre[kListChunk][32];  // slots of the list in lower warps of this tile
  const uint32_t ncls = min(ct.meta[0], ct.cls_bound);
  const uint32_t nmerge = min(ct.meta[2], ct.cls_bound - ncls);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t pos, r, comp;
  const bool live = decode_slot(d, t, tile * kListTile + tid, m, pos, r, comp);
  const uint32_t local = live ? t.sv_local[pos] : 0u;
  const uint32_t* my_row = balg + size_t(tile) * ct.cls_bound * 32;
  uint32_t mask = 0;  // bit cls_lbit[c]: my servant is eligible for class c of its component (merge payload)
  for (uint32_t c0 = 0; c0 < ncls + nmerge; c0 += kListChunk) {
    const uint32_t c1 = min(c0 + kListChunk, ncls + nmerge);
    for (uint32_t i = tid; i < (c1 - c0) * 32; i += kListTile) (&bal[0][0])[i] = my_row[c0 * 32 + i];
    __syncthreads();
    for (uint32_t c = c0 + warp; c < c1; c += 32) {  // exclusive prefix over the warps, per list
      const uint32_t v = __popc(bal[c - c0][lane]);
      uint32_t x = v;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, s);
        if (lane >= s) x += y;
      }
      pre[c - c0][lane] = (uint16_t)(x - v);
    }
    __syncthreads();
    for (uint32_t c = c0; c < c1; ++c) {
      const uint32_t word = bal[c - c0][warp];
      if ((word >> lane) & 1u) {
        if (c < ncls) mask |= 1u << (ct.cls_lbit[c] & 31u);
        const uint32_t dst = offs[c * n_tiles + tile] + pre[c - c0][warp] + __popc(word & ((1u << lane) - 1));
        // class list: (servant, running_tasks value of the slot); pseudo-class: (servant, class mask)
        if (dst < list_cap) list[dst] = make_uint2(local, c < ncls ? r : mask);
        else ct.meta[1] = 1;  // more (class, slot) pairs than provisioned: the host reruns with solver 1
      }
    }
    __syncthreads();  // bal / pre are reused by the next chunk
  }
}

__global__ void __launch_bounds__(kListTile) k_list_fill(const unsigned long long* __restrict__ m_ptr, SlotDecode d,
                                                         TopoView t, ClassTable ct, uint32_t n_tiles,
                                                         const uint32_t* __restrict__ offs,
                                                         const uint32_t* __restrict__ balg,
                                                         uint2* __restrict__ list, uint32_t list_cap) {
  list_fill_tile(blockIdx.x, (uint32_t)*m_ptr, d, t, ct, n_tiles, offs, balg, list, list_cap);
}

}  // namespace yd
