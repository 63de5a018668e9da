// solve_merge.cuh -- the merge solver: the slot-side formulation of the sequential fold,
// chunk-parallel with exact speculation.
//
// The reference decides requests one at a time (task_dispatcher.cc:93-140): request i takes the
// smallest untaken slot (tier, r/cap, position) among its class's eligible servants, skipping
// the first free servant on its own IP ("self", cc:372-379) unless nothing else is free
// (cc:394-396).  Requests rank slots by the common sorted order (own servant's slots last),
// slots "rank" requests by FIFO index: with a common order on one side the stable matching is
// unique and it is what the sequential fold produces.  It can equally be produced from the slot
// side:
//
//     walk the component's slots in sorted order; each slot (s, r) takes the EARLIEST unserved
//     request i among the classes servant s is eligible for, with self(i) != s.
//
// Requests of a class are served in FIFO order except that a slot of servant s passes over
// requests from s itself; those stay "pending" (a handful at most) and are the class's first
// candidates for the next slots.  State = one served-or-passed counter h_c per class + the
// pending set.  The only way this differs from the sequential fold is the last-resort rule: a
// request that ends up unserved although a slot of its own servant went to a LATER request (or
// stayed empty) would have taken that slot.  k_merge_check detects exactly that blocking pair
// after the fact (it needs every class to be running out of slots while the requestor's own
// servant still has one -- the end game of a saturated class); the component is then decided by
// the sequential solver (solve_stream.cuh) instead.  No blocking pair => stable => identical to
// the reference.
//
// Staging (TMA).  A chunk's warp reads three streams: its window of the sorted slot list and, per
// class, the head of the class's FIFO request records.  Both are staged in shared-memory rings of
// four 256-byte blocks filled by `cp.async.bulk` (one elected lane issues, completion is counted on
// an mbarrier): the block a step will need NEXT is requested when the step starts and waited for
// when it ends, so the copy overlaps the step's fixed-point rounds.
//
// One launch.  k_merge_solve is persistent (one warp per block, co-resident grid): the Jacobi rounds,
// the slot -> request scatter and the last-resort check are phases of one kernel separated by a
// grid barrier; it stops as soon as a round re-runs nothing.  A batch without merge components
// costs one empty launch.
//
// Parallelism.  The slot list of a component is cut into chunks of `chunk` slots, one warp each.
// The state at a chunk boundary is not known in advance, so it is GUESSED -- after x slots the
// served requests are (nearly) the first x requests of the component in FIFO order, so h_c = the
// number of class-c requests among those -- and every chunk runs from its guess at once.  Round
// r >= 1 re-runs every chunk whose start state differs from what its predecessor produced in
// round r-1 (Jacobi iteration on the boundary states).  After round r the first r+1 chunks are
// final, so the iteration always ends with the sequential result; it ends after 2-3 rounds when
// a wrong guess "heals" inside a chunk (discrepancies between two trajectories annihilate as
// soon as one slot can serve both affected classes; measured: a few hundred slots).  A round in
// which no chunk re-ran certifies the chain: every start state equals its predecessor's end state.
//
// Inside a chunk the warp takes 32 slots per step.  With three or more classes the CLASSES sit in the
// lanes (lane k holds the head of class k's queue) and the 32 slots are decided one after the other
// by a warp-wide min each; with one or two classes the SLOTS sit in the lanes and iterate
// "recompute my choice given the lanes before me" to the (unique) fixed point.  A slot that would
// serve a request from its own servant ends the step: it -- and every slot while requests are
// pending -- is handled by the exact one-slot step.
#pragma once
#include "classes.cuh"

namespace yd {

// Pending requests are kept as runs: a slot of servant s passes over the CONSECUTIVE requests from s
// at the head of a class queue, i.e. a range [j0, j1) of that queue with one own servant.
constexpr uint32_t kMergePend = 8;         // pending runs a state can carry
constexpr uint32_t kMergeStateWords = 60;  // h[32] | np | pad[3] | pk[8] | pj0[8] | pj1[8]
constexpr uint32_t kMsNp = 32, kMsPk = 36, kMsJ0 = 44, kMsJ1 = 52;
constexpr uint32_t kMergeSkipMax = 1u << 20;  // longest run of own-servant requests walked over (then: sequential solver)
constexpr uint32_t kMergeMaxRounds = 16;   // changed[] is indexed by round & 15

// Why a component was handed back to the sequential solver: MergePlan::viol collects one bit per rule (atomicOr), so the
// solve's debug line can name the rules that fired.  Readers only test it for non-zero.
constexpr uint32_t kBackPend = 1;     // more pending runs than a state carries (kMergePend)
constexpr uint32_t kBackSkip = 2;     // a run of own-servant requests longer than kMergeSkipMax
constexpr uint32_t kBackWindow = 4;   // a record outside the gathered window (range-sharded queue)
constexpr uint32_t kBackCheck = 8;    // a blocking pair: the last-resort rule (k_merge_check)
constexpr uint32_t kBackClasses = 16; // more classes than the rings are provisioned for (cannot happen)
// A chunk whose run met one of the first three ends with this in its end state's np word and the reason in the next:
// its start state may be a wrong guess, so the component is handed back only if the chunk's run is still this one once
// the rounds have settled.
constexpr uint32_t kMergeDead = 0xFFFFFFFFu;

struct MergePlan {
  uint32_t* bar;         // [4] grid barrier arrivals (zeroed with the rest of the scratch region)
  uint32_t* viol;        // [n_comps] kBack* mask, non-zero: the component needs the sequential solver after all
  uint32_t* changed;     // [16] chunks re-run in round r (r & 15)
  uint32_t* dead;        // [16] blocks holding a chunk whose end state is kMergeDead after round r (r & 15)
  uint32_t* tau;         // [S] request index that took the servant's LAST slot (kNone: still free)
};

struct MergeArgs {
  TopoView t;
  ClassTable ct;
  MergePlan mp;
  ServantArrays sv;
  const DynParams* dp;
  const uint32_t* comp_mode;
  const uint32_t* list_off;  // scanned (class-major, tile-minor) list counts
  uint32_t n_list_tiles;
  const uint2* list;         // pseudo-class lists: (servant local index, class mask)
  const uint32_t* rank_off;  // scanned (class-major, tile-minor) request counts
  uint32_t n_rank_tiles;
  const uint2* rq;           // per-class FIFO request lists: (request, own servant or kNone)
  const uint32_t* rcls;      // [n] class of each request
  const uint32_t* rself;     // [n] own servant of each request
  uint32_t* slot_pick;       // [list capacity] request that took the slot, or kNone
  uint32_t* st_in;           // [max_chunks][kMergeStateWords] start state of the chunk's last run
  uint32_t* st_out;          // [max_chunks][kMergeStateWords] end state of the chunk's last run
  uint32_t chunk;            // slots per chunk (multiple of 32)
  uint32_t max_chunks;
  uint32_t kcap;             // classes per component the request rings are provisioned for (<= 32)
  uint32_t rq_blocks;        // whole 32-record blocks in the rq / list allocations (bulk copies stay inside)
  uint32_t ls_blocks;
  uint32_t* res;
  RqLayout L;
  unsigned long long* diag;  // [2] rounds taken, chunks (solver diagnostics, Counters::pad)
};

// ---- mbarrier / bulk-copy (TMA) primitives ------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE%=;\n"
      "bra LAB_WAIT%=;\n"
      "LAB_DONE%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 256 bytes global -> shared, completion counted on `bar` (cp.async.bulk = the TMA engine's 1-D copy).
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

constexpr uint32_t kRingBlocks = 4;               // 32-record blocks per ring
constexpr uint32_t kRingRecs = kRingBlocks * 32;  // ring slot of record x: x & (kRingRecs - 1)

struct MergeSmem {                // static part; the rings are dynamic shared memory
  uint32_t chunk_base[kMaxClasses + 1];
  uint32_t st[kMergeStateWords];
  uint32_t cnt[32];
  uint32_t a[32];                 // per class: absolute rq index of its next record (rq_base + h)
  uint32_t lim[32];               // per class: records at hand from there (window - h)
  uint32_t more[32];              // per class: requests beyond the window exist (sharded queue only)
  uint32_t ovf;
  unsigned long long mbar[33];    // one mbarrier per stream: class k's records (k < 32), the slot list (32)
};


// Boundary guess: h_k = number of class-k requests among the first `x` requests of the component
// (classes without eligible servants do not count: they are EnvironmentNotFound and take nothing).
// Lane k < K owns class k: `cid` its class id, `base` its row start in rank_off, `n` its requests.
__device__ __forceinline__ uint32_t merge_guess(const MergeArgs& a, uint32_t comp, uint32_t K, uint32_t lane,
                                                uint32_t cid, uint32_t base, uint32_t n, uint32_t x,
                                                uint32_t* s_cnt) {
  const uint32_t nrt = a.n_rank_tiles;
  const uint32_t total = __reduce_add_sync(0xffffffffu, lane < K ? n : 0u);
  if (x >= total) return n;
  // F(tile) = component requests in tiles [0, tile); find T with F(T) <= x < F(T + 1), 32 probes per step
  uint32_t lo = 0, hi = nrt;
  while (hi - lo > 1) {
    const uint32_t step = (hi - lo + 31) / 32;
    const uint32_t cand = min(lo + lane * step, hi);
    uint32_t f = 0;
    for (uint32_t k = 0; k < K; ++k) {
      const uint32_t ck = __shfl_sync(0xffffffffu, cid, k), bk = __shfl_sync(0xffffffffu, base, k);
      const uint32_t nk = __shfl_sync(0xffffffffu, n, k);
      if (nk) f += a.rank_off[ck * nrt + cand] - bk;
    }
    const uint32_t okb = __ballot_sync(0xffffffffu, cand < hi && f <= x);  // lane 0 (cand == lo) always qualifies
    const uint32_t j = 31 - __clz(okb);
    const uint32_t nlo = __shfl_sync(0xffffffffu, cand, j);
    const uint32_t nhi = j < 31 ? min(hi, __shfl_sync(0xffffffffu, cand, (j + 1) & 31)) : hi;
    lo = nlo;
    hi = max(nhi, lo + 1);
  }
  const uint32_t T = lo;
  uint32_t before = 0;  // F(T)
  {
    const uint32_t mine = (lane < K && n) ? a.rank_off[cid * nrt + T] - base : 0u;
    before = __reduce_add_sync(0xffffffffu, mine);
  }
  uint32_t h = (lane < K && n) ? a.rank_off[cid * nrt + T] - base : 0u;
  uint32_t need = x - before;  // requests of the component to take from tile T
  s_cnt[lane] = 0;
  __syncwarp();
  const uint32_t nreq = a.dp->n;
  uint32_t cls_v[32];
#pragma unroll
  for (int it = 0; it < 32; ++it) {
    const uint32_t q = T * 1024u + it * 32u + lane;
    cls_v[it] = q < nreq ? __ldg(a.rcls + q) : kNone;
  }
#pragma unroll
  for (int it = 0; it < 32; ++it) {
    if (need == 0) break;
    const uint32_t c = cls_v[it];
    uint32_t lk = kNone;
    if (c != kNone && a.ct.cls_comp[c] == comp && a.ct.cls_nelig[c] != 0) lk = a.ct.cls_lbit[c];
    const uint32_t memb = __ballot_sync(0xffffffffu, lk != kNone);
    const bool valid = lk != kNone && (uint32_t)__popc(memb & ((1u << lane) - 1)) < need;
    const uint32_t peers = __match_any_sync(0xffffffffu, valid ? lk : 64u + lane);
    if (valid && (peers & ((1u << lane) - 1)) == 0) s_cnt[lk & 31u] += __popc(peers);
    need -= min(need, (uint32_t)__popc(memb));
    __syncwarp();
  }
  __syncwarp();
  if (lane < K && n) h = min(n, h + s_cnt[lane]);
  return h;
}

// The same guess when only the class request lists are at hand (range-sharded queue: the tile counts
// of the other ranks are not here, the gathered records are): the threshold T with exactly x records
// q < T over the component's classes, h_k = how many of class k's.  Binary search on T; every lane
// keeps the bracket of its own lower bound, so a step costs a probe or two.
__device__ __forceinline__ uint32_t merge_guess_rq(const MergeArgs& a, uint32_t K, uint32_t lane, uint32_t rq_base,
                                                   uint32_t n, uint32_t win, uint32_t x) {
  const uint32_t have = lane < K ? min(n, win) : 0u;  // records at hand
  if (x >= __reduce_add_sync(0xffffffffu, have)) return lane < K ? n : 0u;
  unsigned long long tlo = 0, thi = 1ull << 32;  // invariant: count(< tlo) <= x < count(< thi) ... searched as "first T with count >= x"
  uint32_t blo = 0, bhi = have;                   // my lower bound for any T in [tlo, thi] lies in [blo, bhi]
  while (thi - tlo > 1) {
    const unsigned long long tm = (tlo + thi) >> 1;
    uint32_t lo = blo, hi = bhi;
    while (lo < hi) {  // first record >= tm
      const uint32_t mid = (lo + hi) >> 1;
      if ((unsigned long long)a.rq[rq_base + mid].x < tm) lo = mid + 1; else hi = mid;
    }
    const uint32_t cnt = __reduce_add_sync(0xffffffffu, lo);
    if (cnt <= x) { tlo = tm; blo = lo; } else { thi = tm; bhi = lo; }
  }
  // count(< tlo) <= x < count(< thi = tlo + 1): records are distinct, so count(< tlo) == x or the record tlo is the x-th;
  // blo is my count of records < tlo
  return blo;
}


// (pseudo-class index, chunk inside the component) of global chunk t.
__device__ __forceinline__ void merge_locate(const MergeSmem& sm, uint32_t nmerge, uint32_t t, uint32_t& midx, uint32_t& b) {
  uint32_t lo = 0, hi = nmerge;  // largest m with chunk_base[m] <= t
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (sm.chunk_base[mid] <= t) lo = mid; else hi = mid;
  }
  midx = lo;
  b = t - sm.chunk_base[lo];
}

__device__ __forceinline__ void merge_grid_sync(uint32_t* bar, uint32_t& epoch, uint32_t lane) {
  __syncwarp();
  ++epoch;
  if (lane == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    const uint32_t want = epoch * gridDim.x;
    while (*reinterpret_cast<volatile uint32_t*>(bar) < want) __nanosleep(32);
    __threadfence();
  }
  __syncwarp();
}

// Runs chunk t in round r.  Returns 1 if it ran (its start state was new), 0 otherwise.
__device__ uint32_t merge_run_chunk(const MergeArgs& a, MergeSmem& sm, uint2* ring_ls, uint2* ring_rq, uint32_t ncls,
                                    uint32_t midx, uint32_t b, uint32_t t, uint32_t r, uint32_t& par_rq, uint32_t& par_ls) {
  const uint32_t lane = threadIdx.x;
  const uint32_t lt_mask = (1u << lane) - 1;
  const uint32_t comp = a.ct.merge_comp[midx];
  if (__ldcg(a.mp.viol + comp)) return 0;
  if (b == 0 && r > 0) return 0;  // the first chunk starts from the true state: final after round 0
  const uint32_t K = a.ct.comp_ncls[comp];
  if (K > a.kcap) {  // (cannot happen: the rings are provisioned for min(32, cls_bound) classes)
    if (lane == 0) atomicOr(a.mp.viol + comp, kBackClasses);
    return 0;
  }
  const uint32_t nrt = a.n_rank_tiles;
  uint32_t cid = 0, rq_base = 0, n = 0, win = 0, h = 0;
  if (lane < K) {
    cid = a.ct.comp_cls[midx * 32 + lane];
    rq_base = a.L.Base(cid);
    n = a.ct.cls_nelig[cid] ? a.L.Gn(cid) : 0u;  // nobody eligible: all ENF already
    win = min(n, a.L.Win(cid));                  // records [0, win) of the class are in rq (one GPU: all of them)
  }
  const uint32_t pc = ncls + midx;
  const uint32_t L0 = a.list_off[pc * a.n_list_tiles], L1 = a.list_off[(pc + 1) * a.n_list_tiles];
  const uint32_t lb = L0 + b * a.chunk, le = min(L1, lb + a.chunk);
  uint32_t* my_in = a.st_in + size_t(t) * kMergeStateWords;
  uint32_t* my_out = a.st_out + size_t(t) * kMergeStateWords;
  uint32_t* st = sm.st;

  // ---- start state -------------------------------------------------------------------------
  if (lane < kMergeStateWords - 32) st[32 + lane] = 0;
  if (lane == 0) sm.ovf = 0;
  __syncwarp();
  if (b == 0) {
    h = 0;
  } else if (r == 0) {
    h = a.L.sharded ? merge_guess_rq(a, K, lane, rq_base, n, win, b * a.chunk)
                    : merge_guess(a, comp, K, lane, cid, lane < K ? a.rank_off[cid * nrt] : 0u, n, b * a.chunk, sm.cnt);
  } else {
    const uint32_t* prev = a.st_out + size_t(t - 1) * kMergeStateWords;
    const uint32_t p0 = __ldcg(prev + lane);
    const uint32_t p1 = lane < kMergeStateWords - 32 ? __ldcg(prev + 32 + lane) : 0u;
    const uint32_t m0 = my_in[lane];
    const uint32_t m1 = lane < kMergeStateWords - 32 ? my_in[32 + lane] : 0u;
    if (__all_sync(0xffffffffu, p0 == m0 && p1 == m1)) return 0;  // consistent with my predecessor: nothing to do
    if (__shfl_sync(0xffffffffu, p1, 0) == kMergeDead) return 0;  // nothing to start from (see kMergeDead)
    h = lane < K ? min(p0, n) : 0u;
    if (lane < kMergeStateWords - 32) st[32 + lane] = p1;
    __syncwarp();
    if (lane == 0) st[kMsNp] = min(st[kMsNp], kMergePend);
    __syncwarp();
  }
  my_in[lane] = lane < K ? h : 0u;
  if (lane < kMergeStateWords - 32) my_in[32 + lane] = st[32 + lane];
  uint32_t np = st[kMsNp];

  // ---- the chunk's slots -----------------------------------------------------------------------
  uint64_t* mbar = reinterpret_cast<uint64_t*>(sm.mbar);
  uint32_t base = lb;
  uint32_t dead = 0;  // kBack* reasons to hand the component back
  // Ring bookkeeping, per stream owner (lane k for class k's records, lane 0 also for the slot list): blocks below
  // `*_hi` are in the ring or on their way, blocks below `*_ok` have landed.  A step reads blocks jb and jb + 1 of a
  // stream; block jb + 2 is requested as soon as jb is reached, i.e. a whole block of progress before it is read,
  // and nobody waits for it until then.  Every stream has its OWN mbarrier (one request in flight per stream), so a
  // class that crosses a block boundary never waits for another class's copy: steady-state steps touch neither a
  // barrier nor HBM.
  uint32_t rq_hi = 0, rq_ok = 0, ls_hi = 0, ls_ok = 0;
  bool prime = true;          // the rings hold nothing useful (chunk start, or a one-slot step moved h)
  bool rq_pend = false, ls_pend = false;
  uint32_t rq_par = par_rq, ls_par = par_ls;  // phase parity of my barriers (kept across chunks by the caller)
  while (base < le) {
    if (np == 0 && __reduce_add_sync(0xffffffffu, lane < K ? n - h : 0u) == 0) break;  // every request is served
    // ---- top up the rings ---------------------------------------------------------------------------------
    {
      const uint32_t jb = (rq_base + h) >> 5;
      const bool mine = lane < K && h < win;
      if (mine && (prime || rq_hi < jb || rq_hi > jb + 3)) { rq_hi = jb; rq_ok = jb; }  // nothing useful there
      const bool need = mine && rq_hi < jb + 3;
      const uint32_t ljb = base >> 5;
      if (lane == 0 && (prime || ls_hi < ljb || ls_hi > ljb + 3)) { ls_hi = ljb; ls_ok = ljb; }
      const bool lneed = lane == 0 && ls_hi < ljb + 3;
      if (__any_sync(0xffffffffu, need || lneed)) {
        // my previous request (a block of progress ago) must have landed before the stream's barrier is reused
        if (need && rq_pend) { mbar_wait(&mbar[lane], rq_par); rq_par ^= 1; rq_pend = false; rq_ok = rq_hi; }
        if (lneed && ls_pend) { mbar_wait(&mbar[32], ls_par); ls_par ^= 1; ls_pend = false; ls_ok = ls_hi; }
        __syncwarp();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic reads of a slot before its refill
        const uint32_t needb = __ballot_sync(0xffffffffu, need);
        for (uint32_t todo = needb; todo; todo &= todo - 1) {
          const uint32_t k = __ffs(todo) - 1;
          const uint32_t f = __shfl_sync(0xffffffffu, rq_hi, k), e2 = __shfl_sync(0xffffffffu, jb + 3, k);
          if (lane == 0) {
            uint32_t bytes = 0;
            for (uint32_t blk = f; blk < e2; ++blk) {
              if (blk >= a.rq_blocks) break;
              bulk_g2s(ring_rq + size_t(k) * kRingRecs + (blk & (kRingBlocks - 1)) * 32, a.rq + size_t(blk) * 32, 256, &mbar[k]);
              bytes += 256;
            }
            mbar_arrive_expect_tx(&mbar[k], bytes);
          }
        }
        if (__shfl_sync(0xffffffffu, lneed ? 1u : 0u, 0)) {
          if (lane == 0) {
            uint32_t bytes = 0;
            for (uint32_t blk = ls_hi; blk < ljb + 3; ++blk) {
              if (blk >= a.ls_blocks) break;
              bulk_g2s(ring_ls + (blk & (kRingBlocks - 1)) * 32, a.list + size_t(blk) * 32, 256, &mbar[32]);
              bytes += 256;
            }
            mbar_arrive_expect_tx(&mbar[32], bytes);
            ls_hi = ljb + 3;
            ls_pend = true;
          }
        }
        if (need) { rq_hi = jb + 3; rq_pend = true; }
        __syncwarp();
      }
      // this step reads blocks jb, jb + 1 of every stream: have they landed?
      if (mine && rq_ok < jb + 2 && rq_pend) { mbar_wait(&mbar[lane], rq_par); rq_par ^= 1; rq_pend = false; rq_ok = rq_hi; }
      if (lane == 0 && ls_ok < ljb + 2 && ls_pend) { mbar_wait(&mbar[32], ls_par); ls_par ^= 1; ls_pend = false; ls_ok = ls_hi; }
      __syncwarp();
      prime = false;
    }

    if (np == 0) {
      const uint32_t idx = base + lane;
      const uint2 e = idx < le ? ring_ls[idx & (kRingRecs - 1)] : make_uint2(0, 0);  // mask 0: no slot in this lane
      uint32_t fb = 32, my_pick = kNone;
      if (K > 2) {
        // Slot by slot, the CLASSES in the lanes: lane k holds the head of class k's queue (`cur`, and the record
        // behind it) and a bit per slot "my class is eligible on that slot's servant"; a slot's verdict is one
        // warp-wide min over those heads.  The loop carries one dependency -- the winner's head moves on -- through a
        // redux and a handful of ALU instructions; no votes, no shuffles, no branches inside.
        constexpr uint32_t kMissing = 0xFFFFFFFEu;  // "a request exists here but its record was not gathered" (sharded queue)
        const uint32_t my_a = rq_base + h, my_lim = (lane < K && win > h) ? win - h : 0u;
        const uint32_t my_more = (lane < K && n > win) ? n - h : 0u;
        const uint2* my_ring = ring_rq + size_t(lane < K ? lane : 0) * kRingRecs;
        uint32_t elig = 0;  // bit j: slot j's servant is eligible for my class
        for (uint32_t k = 0; k < K; ++k) {
          const uint32_t bk = __ballot_sync(0xffffffffu, (e.y >> k) & 1u);
          if (lane == k) elig = bk;
        }
        auto rec = [&](uint32_t i) -> uint2 {  // my class's i-th record from h
          if (i < my_lim) return my_ring[(my_a + i) & (kRingRecs - 1)];
          return make_uint2(i < my_more ? kMissing : kNone, kNone);
        };
        uint32_t taken = 0;
        bool miss = false;
        uint2 cur = rec(0), nxt = rec(1);
#pragma unroll 4
        for (int j = 0; j < 32; ++j) {
          const bool in = (elig >> j) & 1u;
          const uint32_t cand = in ? cur.x : kNone;
          miss |= in && cur.x == kMissing;  // whoever wins this slot, an unseen request might have been earlier
          const uint32_t m = __reduce_min_sync(0xffffffffu, cand);
          const bool won = in && cand == m;  // (m == kNone: nobody is `in` with a request left; harmless below)
          if (lane == (uint32_t)j) my_pick = m;
          if (won && m < kMissing) {
            sm.a[j] = cur.y;    // the served request's own servant ...
            sm.lim[j] = lane;   // ... and its class, for the check after the loop
            ++taken;
            cur = nxt;
            nxt = rec(taken + 1);
          }
        }
        __syncwarp();
        if (__any_sync(0xffffffffu, miss)) { dead = kBackWindow; break; }
        // a slot that took a request from its own servant: the step ends before it (the one-slot step decides it)
        const uint32_t cb = __ballot_sync(0xffffffffu, my_pick != kNone && sm.a[lane] == e.x);
        if (cb) {
          fb = (uint32_t)__ffs(cb) - 1u;
          const uint32_t pc_ = (my_pick != kNone && lane < fb) ? sm.lim[lane] : 32u;  // class of the request my slot took
          taken = 0;
          for (uint32_t k = 0; k < K; ++k) {
            const uint32_t tk = __popc(__ballot_sync(0xffffffffu, pc_ == k));
            if (lane == k) taken = tk;
          }
        }
        h += taken;
      } else {
      if (lane < K) { sm.a[lane] = rq_base + h; sm.lim[lane] = win > h ? win - h : 0u; sm.more[lane] = n > win ? n - h : 0u; }
      __syncwarp();
      uint32_t pick = 32, best = kNone, bself = kNone;
      for (int round = 0; round < 33; ++round) {
        uint32_t npick = 32, nbest = kNone, nself = kNone;
        for (uint32_t k = 0; k < K; ++k) {
          const uint32_t cnt = __popc(__ballot_sync(0xffffffffu, pick == k) & lt_mask);  // earlier slots on class k
          if ((e.y >> k) & 1u) {
            if (cnt < sm.lim[k]) {
              const uint2 v = ring_rq[size_t(k) * kRingRecs + ((sm.a[k] + cnt) & (kRingRecs - 1))];
              if (v.x < nbest) { nbest = v.x; npick = k; nself = v.y; }
            } else if (cnt < sm.more[k]) {
              sm.ovf = kBackWindow;  // a request whose record was not gathered (sharded queue only)
            }
          }
        }
        const bool moved = npick != pick;
        pick = npick; best = nbest; bself = nself;
        if (!__any_sync(0xffffffffu, moved)) break;
      }
      __syncwarp();
      if (sm.ovf) { dead = sm.ovf; break; }
      // a lane that would serve a request from its own servant: commit the lanes before it only
      const uint32_t cb = __ballot_sync(0xffffffffu, pick < 32 && bself == e.x);
      fb = cb ? (uint32_t)__ffs(cb) - 1u : 32u;
      for (uint32_t k = 0; k < K; ++k) {
        const uint32_t took = __popc(__ballot_sync(0xffffffffu, lane < fb && pick == k));
        if (lane == k) h += took;
      }
      my_pick = pick < 32 ? best : kNone;
      }
      if (lane < fb && idx < le) a.slot_pick[idx] = my_pick;
      __syncwarp();
      base += fb;
      if (fb == 32) continue;
      if (base >= le) break;
    }
    // ---- one slot, exactly: pending requests first, own-servant requests passed over -----------------
    {
      prime = true;  // h may jump: refill the rings before the next step
      const uint2 e = a.list[base];
      const uint32_t s = e.x;
      uint32_t cq = kNone, cj = 0, pidx = kNone;
      uint32_t ovf = 0;
      if (lane < K && ((e.y >> lane) & 1u)) {
        for (uint32_t p = 0; p < np; ++p) {  // runs of a class are in queue order: the first match is the earliest
          const uint32_t pk = st[kMsPk + p];
          if ((pk >> 24) == lane && (pk & 0xFFFFFFu) != s) {
            if (st[kMsJ0 + p] >= win) { ovf = kBackWindow; break; }
            cq = a.rq[rq_base + st[kMsJ0 + p]].x; pidx = p; break;
          }
        }
        if (pidx == kNone && !ovf) {
          uint32_t j = h;
          while (j < n) {
            if (j >= win) { ovf = kBackWindow; break; }
            const uint2 v = a.rq[rq_base + j];
            if (v.y != s) { cq = v.x; break; }
            ++j;
            if (j - h > kMergeSkipMax) { ovf = kBackSkip; break; }
          }
          cj = j;
        }
      }
      dead = __reduce_or_sync(0xffffffffu, ovf);
      if (dead) break;
      const uint32_t m = __reduce_min_sync(0xffffffffu, cq);
      if (m != kNone) {
        const uint32_t wl = (uint32_t)__ffs(__ballot_sync(0xffffffffu, cq == m)) - 1u;
        if (lane == wl) {
          uint32_t cur = st[kMsNp];
          if (pidx != kNone) {
            if (++st[kMsJ0 + pidx] == st[kMsJ1 + pidx]) {  // the run is used up
              for (uint32_t p = pidx; p + 1 < cur; ++p) {
                st[kMsPk + p] = st[kMsPk + p + 1]; st[kMsJ0 + p] = st[kMsJ0 + p + 1]; st[kMsJ1 + p] = st[kMsJ1 + p + 1];
              }
              --cur;
              st[kMsPk + cur] = 0; st[kMsJ0 + cur] = 0; st[kMsJ1 + cur] = 0;
            }
          } else {
            if (cj > h) {  // [h, cj) are from servant s itself: they wait for another servant's slot
              const uint32_t key = (lane << 24) | (s & 0xFFFFFFu);
              uint32_t last = kNone;  // my class's latest run
              for (uint32_t p = 0; p < cur; ++p) {
                if ((st[kMsPk + p] >> 24) == lane) last = p;
              }
              if (last != kNone && st[kMsPk + last] == key && st[kMsJ1 + last] == h) {
                st[kMsJ1 + last] = cj;  // contiguous with it: one run
              } else if (cur < kMergePend) {
                st[kMsPk + cur] = key; st[kMsJ0 + cur] = h; st[kMsJ1 + cur] = cj;
                ++cur;
              } else {
                sm.ovf = kBackPend;
              }
            }
            h = cj + 1;
          }
          st[kMsNp] = cur;
        }
        __syncwarp();
        if (sm.ovf) { dead = sm.ovf; break; }
        np = st[kMsNp];
      }
      if (lane == 0) a.slot_pick[base] = m;
      base += 1;
    }
  }
  // nothing may still be landing in the rings when the warp moves on
  if (rq_pend) { mbar_wait(&mbar[lane], rq_par); rq_par ^= 1; }
  if (ls_pend) { mbar_wait(&mbar[32], ls_par); ls_par ^= 1; }
  par_rq = rq_par; par_ls = ls_par;
  __syncwarp();
  if (dead) {  // more pending runs than a state carries / a record that was not gathered: the sequential solver decides
    my_out[lane] = 0;
    if (lane < kMergeStateWords - 32) my_out[32 + lane] = lane == 0 ? kMergeDead : lane == 1 ? dead : 0u;
    return 1;
  }
  for (uint32_t idx = base + lane; idx < le; idx += 32) a.slot_pick[idx] = kNone;
  my_out[lane] = lane < K ? h : 0u;
  __syncwarp();
  if (lane < kMergeStateWords - 32) my_out[32 + lane] = st[32 + lane];
  return 1;
}

// The whole merge solver: plan, Jacobi rounds until a round re-runs nothing, slots -> requests, last-resort check.
__global__ void __launch_bounds__(32) k_merge_solve(MergeArgs a) {
  extern __shared__ __align__(16) unsigned char merge_dyn[];
  __shared__ MergeSmem sm;
  uint2* ring_ls = reinterpret_cast<uint2*>(merge_dyn);
  uint2* ring_rq = ring_ls + kRingRecs;
  const uint32_t lane = threadIdx.x;
  if (a.ct.meta[1]) return;
  const uint32_t ncls = min(a.ct.meta[0], a.ct.cls_bound);
  const uint32_t nmerge = min(a.ct.meta[2], a.ct.cls_bound - ncls);
  if (nmerge == 0) return;
  // ---- plan: chunks per merge component (every block computes the same table) --------------------------------
  uint32_t carry = 0;
  for (uint32_t m0 = 0; m0 < nmerge; m0 += 32) {
    const uint32_t m = m0 + lane;
    uint32_t nch = 0;
    if (m < nmerge) {
      const uint32_t pc = ncls + m;
      const uint32_t len = a.list_off[(pc + 1) * a.n_list_tiles] - a.list_off[pc * a.n_list_tiles];
      nch = (len + a.chunk - 1) / a.chunk;
    }
    uint32_t x = nch;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (m < nmerge) sm.chunk_base[m] = carry + x - nch;
    carry += __shfl_sync(0xffffffffu, x, 31);
  }
  const uint32_t total = min(carry, a.max_chunks);
  if (lane == 0) sm.chunk_base[nmerge] = carry;
  mbar_init(reinterpret_cast<uint64_t*>(sm.mbar) + lane, 1);  // one arrival per phase: the elected lane's expect_tx
  if (lane == 0) mbar_init(reinterpret_cast<uint64_t*>(sm.mbar) + 32, 1);
  __syncwarp();
  if (total == 0) return;
  uint32_t par_rq = 0, par_ls = 0, epoch = 0;
  // ---- rounds -----------------------------------------------------------------------------------------------
  for (uint32_t r = 0;; ++r) {
    if (blockIdx.x == 0 && lane == 0) {  // (nobody touches these cells during round r)
      atomicExch(&a.mp.changed[(r + 1) & 15u], 0u);
      atomicExch(&a.mp.dead[(r + 1) & 15u], 0u);
    }
    uint32_t ran = 0;
    for (uint32_t t = blockIdx.x; t < total; t += gridDim.x) {
      uint32_t midx, b;
      merge_locate(sm, nmerge, t, midx, b);
      ran += merge_run_chunk(a, sm, ring_ls, ring_rq, ncls, midx, b, t, r, par_rq, par_ls);
      __syncwarp();
    }
    if (r > 0 && ran && lane == 0) atomicAdd(&a.mp.changed[r & 15u], ran);
    // (only read after a round that re-ran nothing, in which no end state changes)
    if (lane == 0) {
      bool dead = false;
      for (uint32_t t = blockIdx.x; t < total && !dead; t += gridDim.x) dead = __ldcg(a.st_out + size_t(t) * kMergeStateWords + kMsNp) == kMergeDead;
      if (dead) atomicAdd(&a.mp.dead[r & 15u], 1u);
    }
    merge_grid_sync(a.mp.bar, epoch, lane);
    if (r > 0 && atomicAdd(&a.mp.changed[r & 15u], 0u) == 0) {  // nothing re-ran: every start state equals its predecessor's end
      if (blockIdx.x == 0 && lane == 0 && a.diag) { a.diag[0] = r + 1; a.diag[1] = total; }
      if (atomicAdd(&a.mp.dead[r & 15u], 0u)) {
        // the settled chain holds chunks that could not decide their slots (the first of them started from the true
        // state): their components go to the sequential solver
        for (uint32_t t = blockIdx.x; t < total && lane == 0; t += gridDim.x) {
          const uint32_t* out = a.st_out + size_t(t) * kMergeStateWords;
          if (__ldcg(out + kMsNp) != kMergeDead) continue;
          uint32_t midx, b;
          merge_locate(sm, nmerge, t, midx, b);
          atomicOr(a.mp.viol + a.ct.merge_comp[midx], __ldcg(out + kMsNp + 1));
        }
        merge_grid_sync(a.mp.bar, epoch, lane);
      }
      break;
    }
    if (r > total + 2) {  // (cannot happen: after round r the first r + 1 chunks are final)
      if (blockIdx.x == 0 && lane == 0) a.ct.meta[1] = 3;
      return;
    }
  }
  // ---- slots -> requests: verdicts and the take time of every servant's last slot ----------------------------------
  for (uint32_t t = blockIdx.x; t < total; t += gridDim.x) {
    uint32_t midx, b;
    merge_locate(sm, nmerge, t, midx, b);
    const uint32_t comp = a.ct.merge_comp[midx];
    if (__ldcg(a.mp.viol + comp)) continue;
    const uint32_t pc = ncls + midx;
    const uint32_t L0 = a.list_off[pc * a.n_list_tiles], L1 = a.list_off[(pc + 1) * a.n_list_tiles];
    const uint32_t lb = L0 + b * a.chunk, le = min(L1, lb + a.chunk);
    const uint32_t sv_begin = a.t.comp_sv_off[comp];
    for (uint32_t idx = lb + lane; idx < le; idx += 32) {
      const uint32_t q = a.slot_pick[idx];
      const uint32_t li = sv_begin + a.list[idx].x;
      atomicMax(&a.mp.tau[a.t.comp_sv[li]], q);  // slots of one servant are taken in order: the max is its last slot's
      if (q != kNone && q - a.L.q_base < a.L.n_local) a.res[q - a.L.q_base] = li;  // (requests of this rank's range)
    }
  }
}

// The last-resort rule (cc:394-396): an unserved request whose own servant still had a slot at its turn would have
// taken it.  One such request and the component goes to the sequential solver.  (Its own launch: it is a pass over
// all REQUESTS, far wider than the merge kernel's co-resident grid.)
__global__ void __launch_bounds__(256) k_merge_check(MergeArgs a) {
  if (a.ct.meta[1] || a.ct.meta[2] == 0) return;
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= a.dp->n) return;
  const uint32_t c = a.rcls[q];
  if (c == kNone) return;
  const uint32_t comp = a.ct.cls_comp[c];
  if (a.comp_mode[comp] != 2 || !(a.ct.comp_flags[comp] & 1u)) return;
  const uint32_t self = a.rself[q];
  if (self == kNone || a.res[q] != kResTimeout) return;
  const uint32_t pos = a.t.comp_sv[a.t.comp_sv_off[comp] + self];
  if (a.mp.tau[pos] <= a.L.q_base + q) return;  // every slot of the own servant went to an earlier request
  if (a.sv.max_tasks[pos] != 0 && (uint32_t)a.sv.version[pos] >= a.ct.cls_mv[c] && servant_has_env(a.t, pos, a.ct.cls_env[c])) {
    atomicOr(a.mp.viol + comp, kBackCheck);
  }
}

}  // namespace yd
