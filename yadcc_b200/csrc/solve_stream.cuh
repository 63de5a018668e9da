// solve_stream.cuh -- the slot-stream assignment solver (solver 2).
//
// Observation (DESIGN.md "slot streams"): for fixed heartbeat facts the pick key
// of servant s at running_tasks r, (tier, r/cap, position), is STATIC and strictly
// increasing in r, and a servant is free exactly on a prefix of r values.  So the
// reference's per-request arg-min over servants (task_dispatcher.cc:417-451) always
// returns the globally smallest *untaken slot* (s, r) among the request's eligible
// servants.  With all slots sorted once per solve (radix.cuh) and filtered per class
// (classes.cuh), a decision is: walk the class's list from its front pointer, skip
// slots already taken (r < running_tasks[s]) and the requestor's own servant, take
// the first one left; fall back to the own servant's head slot; else Timeout.
// O(1) amortised per decision instead of O(servants).
//
// One CTA per component.  Producer warps stream/filter/compact the request queue
// exactly as in solve_rowscan.cuh; ONE solver warp makes the decisions, up to 32
// per step (speculate-and-commit, see below), falling back to an exact one-request
// walk (32 list entries per step: one coalesced 256-byte load, one shared-memory
// gather of running_tasks, three ballots) for the first request that does not fit.
// running_tasks of the component lives in shared memory for the whole solve.
#pragma once
#include "classes.cuh"
#include "solve_rowscan.cuh"  // bar_sync / bar_arrive, tile constants

namespace yd {

struct StreamArgs {
  const yd_task_req* reqs;
  const DynParams* dp;  // dp->n requests
  uint32_t* res;
  TopoView t;
  ClassTable ct;
  ServantArrays sv;
  const uint32_t* row_len;    // free slots per servant (this solve), or with static_rows: its free_end
  uint32_t static_rows;
  const uint32_t* list_off;   // [n_classes * n_list_tiles + 1] scanned counts; class c starts at list_off[c * n_list_tiles]
  uint32_t n_list_tiles;
  const uint2* list;          // (servant local index, running_tasks value of the slot)
  uint32_t max_comp_servants; // dynamic shared memory holds 2 x this many u32; a larger component keeps its
  uint32_t* gscratch;         // running_tasks copy in HBM/L2 instead: gscratch[2 * S], [comp_sv_off .. ) per component
  uint32_t n_servants;
  const uint32_t* comp_mode;  // [C] 0 = this kernel, 1 = handled by the parallel path, 2 = merge solver ...
  const uint32_t* viol;       // [C] ... unless it handed the component back (solve_merge.cuh)
  Counters* counters;         // pad[0..3]: speculation steps, lanes committed by them, exact walks, walk windows
};

struct StreamShared {
  uint4 desc[2][kTile];  // {request index, class id, self info, -}
  uint32_t cnt[2];
  uint32_t pcnt[2][32];
  uint32_t front[kMaxClasses];  // list index of the first entry not known to be taken
  uint32_t end[kMaxClasses];
  uint8_t fail[kMaxClasses];    // 0 unknown, 1 Timeout for good, 2 EnvironmentNotFound
};

__device__ __forceinline__ uint32_t stream_fail_res(uint8_t f) { return f == 1 ? kResTimeout : kResEnvNotFound; }

// Same two-pass order-preserving compaction as produce_tile, with the class id
// resolved through the class table.
__device__ __forceinline__ void produce_tile_stream(const StreamArgs& a, StreamShared& sh, uint32_t comp,
                                                    uint32_t buf, uint32_t base, uint32_t tile_end, uint32_t gw,
                                                    uint32_t gn, uint32_t lane) {
  const uint32_t chunk = ((kTile + gn - 1) / gn + 31) & ~31u;
  const uint32_t c0 = min(tile_end, base + gw * chunk), c1 = min(tile_end, c0 + chunk);
  uint32_t minebits = 0, my_count = 0, it = 0;
  uint32_t cls_keep[4];  // class ids of my (up to 4 x 32) requests when gn == 8; recomputed otherwise
#pragma unroll
  for (int k = 0; k < 4; ++k) cls_keep[k] = kNone;
  for (uint32_t q0 = c0; q0 < c1; q0 += 32, ++it) {
    const uint32_t q = q0 + lane;
    bool mine = false;
    uint32_t cls = kNone;
    if (q < c1) {
      const uint2 w0 = __ldg(reinterpret_cast<const uint2*>(a.reqs + q));
      const uint32_t env = w0.x, mv = w0.y;
      if (env < a.t.n_envs && __ldg(a.t.env_comp + env) == comp) {
        const uint32_t slot = cls_find(a.ct.keys, ((unsigned long long)env << 32) | mv);
        cls = slot != kNone ? a.ct.slot_cls[slot] : kNone;
        if (cls != kNone) {
          const uint8_t f = sh.fail[cls];
          if (f) a.res[q] = stream_fail_res(f);
          else mine = true;
        }
      }
    }
    if (it < 4) cls_keep[it] = cls;
    minebits |= (mine ? 1u : 0u) << it;
    my_count += __popc(__ballot_sync(0xffffffffu, mine));
  }
  if (lane == 0) sh.pcnt[buf][gw] = my_count;
  bar_sync(kBarProducer, gn * 32);
  uint32_t woff = 0;
  for (uint32_t w = 0; w < gw; ++w) woff += sh.pcnt[buf][w];
  it = 0;
  for (uint32_t q0 = c0; q0 < c1; q0 += 32, ++it) {
    const uint32_t q = q0 + lane;
    const bool mine = (minebits >> it) & 1u;
    const uint32_t bal = __ballot_sync(0xffffffffu, mine);
    if (mine) {
      const uint2* rp = reinterpret_cast<const uint2*>(a.reqs + q);
      uint32_t cls;
      if (it < 4) {
        cls = cls_keep[it];
      } else {
        const uint2 w0 = __ldg(rp);
        cls = a.ct.slot_cls[cls_find(a.ct.keys, ((unsigned long long)w0.x << 32) | w0.y)];
      }
      const uint32_t ip = __ldg(rp + 1).x;
      uint32_t selfinfo = kNone;
      if (ip < a.t.n_ips) {
        uint32_t b = __ldg(a.t.ip_off + ip), e = __ldg(a.t.ip_off + ip + 1);
        if (e - b == 1) {
          uint32_t p = __ldg(a.t.ip_sv + b);
          if (__ldg(a.t.sv_comp + p) == comp) selfinfo = __ldg(a.t.sv_local + p);
        } else if (e - b > 1) {
          selfinfo = 0x80000000u | ip;
        }
      }
      sh.desc[buf][woff + __popc(bal & ((1u << lane) - 1))] = make_uint4(q, cls, selfinfo, 0u);
    }
    woff += __popc(bal);
  }
}

// Position of the (k+1)-th set bit of `m` (k = 0 .. 31), or 32 if m has fewer set bits.
// Five popc steps instead of the software loop behind __fns.
__device__ __forceinline__ uint32_t kth_set_bit(uint32_t m, uint32_t k) {
  if (__popc(m) <= (int)k) return 32;
  uint32_t pos = 0;
#pragma unroll
  for (int w = 16; w >= 1; w >>= 1) {
    const uint32_t lowmask = (1u << w) - 1;
    const uint32_t cnt = __popc((m >> pos) & lowmask);
    if (k >= cnt) { k -= cnt; pos += w; }
  }
  return pos;
}

constexpr int kStreamProducers = 8;

__global__ void __launch_bounds__((kStreamProducers + 1) * 32, 1) k_solve_stream(StreamArgs a) {
  extern __shared__ uint32_t dyn_smem[];  // run_s[max_comp_servants], lim_s[max_comp_servants]
  __shared__ StreamShared sh;
  const uint32_t comp = blockIdx.x;
  if (a.ct.meta[1]) return;  // class table overflow: the host reruns this batch with the row-scan solver
  const uint32_t mode = a.comp_mode[comp];
  if ((mode != 0 && !(mode == 2 && a.viol[comp])) || a.ct.comp_ncls[comp] == 0) return;  // nothing (for us) to do
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t nall = (kStreamProducers + 1) * 32;
  const uint32_t sv_begin = a.t.comp_sv_off[comp];
  const uint32_t n_sv = a.t.comp_sv_off[comp + 1] - sv_begin;
  // running_tasks of the component for the whole solve: shared memory, or (components beyond what it holds --
  // tens of thousands of servants behind one digest) a per-component slice of an HBM scratch array, L2-resident
  const bool big = n_sv > a.max_comp_servants;
  uint32_t* run_s = big ? a.gscratch + sv_begin : dyn_smem;
  uint32_t* lim_s = big ? a.gscratch + a.n_servants + sv_begin : dyn_smem + a.max_comp_servants;  // first value at which the servant is full

  const uint32_t n_cls = a.ct.meta[0];
  for (uint32_t c = tid; c < kMaxClasses; c += nall) {
    uint32_t f = 0, fr = 0, en = 0;
    if (c < n_cls && a.ct.cls_comp[c] == comp) {
      fr = a.list_off[c * a.n_list_tiles];
      en = a.list_off[(c + 1) * a.n_list_tiles];
      if (a.ct.cls_nelig[c] == 0) f = 2;  // nobody eligible: EnvironmentNotFound, statically
    }
    sh.front[c] = fr; sh.end[c] = en; sh.fail[c] = (uint8_t)f;
  }
  for (uint32_t i = tid; i < n_sv; i += nall) {
    const uint32_t pos = a.t.comp_sv[sv_begin + i];
    const uint32_t r0 = a.sv.run[pos];
    run_s[i] = r0;
    lim_s[i] = a.static_rows ? max(r0, a.row_len[pos]) : r0 + a.row_len[pos];
  }
  __syncthreads();

  const uint32_t n_req = a.dp->n;
  const uint32_t n_tiles = (n_req + kTile - 1) / kTile;
  // ======================= producer warps (1..8) ==============================
  if (warp >= 1) {
    const uint32_t pw = warp - 1;
    for (uint32_t t = 0; t < n_tiles; ++t) {
      const uint32_t buf = t & 1, base = t * kTile, tile_end = min(n_req, base + kTile);
      if (t >= 2) bar_sync(kBarFree0 + buf, nall);
      produce_tile_stream(a, sh, comp, buf, base, tile_end, pw, kStreamProducers, lane);
      if (pw == 0 && lane == 0) {
        uint32_t c = 0;
        for (uint32_t w = 0; w < kStreamProducers; ++w) c += sh.pcnt[buf][w];
        sh.cnt[buf] = c;
      }
      __threadfence_block();
      bar_arrive(kBarFull0 + buf, nall);
    }
    return;
  }

  // ======================= the solver warp ======================================
  // Up to 32 consecutive requests are decided per step.  Lane i speculates that the
  // sequential fold would hand it entry front[class] + (its rank among the group's
  // earlier requests of the same class); that is exactly right iff
  //   (1) that entry and those of all lower-ranked same-class lanes are untaken and not the
  //       respective requestor's own servant (nobody skips anything), and
  //   (2) no earlier lane of ANOTHER class claims the same slot (s, r).
  // [Why (2) suffices: a slot of s can only be passed over once it is taken, and slots of
  // one servant are taken in r order, so any interference between classes shows up as two
  // lanes claiming the same (s, r).]  The longest prefix of lanes satisfying (1)-(2) is
  // committed at once; the first offender is decided by the exact one-request walk below,
  // and the next step starts after it.
  // Speculation is adaptive: when other classes keep consuming the slots at a class's
  // front (heavily shared servants), groups commit one or two lanes and the attempt is
  // pure overhead; after a short commit the next `cooldown` requests go straight to the
  // exact walk.
  const uint32_t lt_mask = (1u << lane) - 1;
  uint32_t cooldown = 0;
  unsigned long long st_steps = 0, st_lanes = 0, st_walks = 0, st_windows = 0;
  for (uint32_t t = 0; t < n_tiles; ++t) {
    const uint32_t buf = t & 1;
    bar_sync(kBarFull0 + buf, nall);
    const uint32_t cnt = sh.cnt[buf];
    const uint4* __restrict__ dl = sh.desc[buf];
    uint32_t at = 0;
    while (at < cnt) {
      if (cooldown == 0) {
        const uint32_t g = min(32u, cnt - at);
        const bool act = lane < g;
        const uint32_t act_mask = g == 32 ? 0xffffffffu : ((1u << g) - 1);
        const uint4 ds = act ? dl[at + lane] : make_uint4(0, kNone, kNone, 0);
        const uint32_t c = ds.y;
        const uint32_t c0 = __shfl_sync(0xffffffffu, c, 0);
        const bool one_class = __all_sync(0xffffffffu, !act || c == c0);
        const bool multi_self = ds.z != kNone && (ds.z & 0x80000000u);  // several own servants: exact path
        bool ok = act;
        uint2 e = make_uint2(kNone, lane);
        bool has_slot = false;
        uint32_t win_pos = 0, peers = act_mask, rank = lane;
        uint8_t f;
        if (one_class) {
          // All lanes of one class (the common shape: one dominant compiler): look at the 32
          // list entries from the front together and hand the k-th UNTAKEN one to the lane of
          // rank k -- tolerant of slots other classes consumed since the front last moved.
          f = sh.fail[c0];
          const uint32_t idx = sh.front[c0] + lane;
          uint2 w = make_uint2(0, 0);
          const bool valid = !f && idx < sh.end[c0];
          if (valid) w = a.list[idx];
          const uint32_t U = __ballot_sync(0xffffffffu, valid && !(w.y < run_s[w.x]));
          const uint32_t p = kth_set_bit(U, lane);  // 32 if there are not that many
          const uint32_t src = p & 31;
          const uint32_t ex = __shfl_sync(0xffffffffu, w.x, src), ey = __shfl_sync(0xffffffffu, w.y, src);
          if (act && !f) {
            ok = p < 32 && !multi_self && ex != ds.z;  // got one, and it is not my own servant
            if (ok) { e = make_uint2(ex, ey); has_slot = true; win_pos = p; }
          }
          if (__ballot_sync(0xffffffffu, act && !ok) & lt_mask) ok = false;  // (1): lower ranks must be clean
        } else {
          f = act ? sh.fail[c] : (uint8_t)0;
          peers = __match_any_sync(0xffffffffu, c);  // inactive lanes share class kNone
          rank = __popc(peers & lt_mask);
          if (act && !f) {
            const uint32_t idx = sh.front[c] + rank;
            ok = idx < sh.end[c] && !multi_self;
            if (ok) {
              e = a.list[idx];
              ok = !(e.y < run_s[e.x]) && e.x != ds.z;  // untaken, and not my own servant
              has_slot = ok;
              if (!ok) e = make_uint2(kNone, lane);
            }
          }
          const uint32_t okb = __ballot_sync(0xffffffffu, ok);
          if (peers & lt_mask & ~okb) ok = false;  // (1): a lower-ranked lane of my class broke the pattern
          // (2): an earlier lane of another class owns that very slot
          const unsigned long long slot = ((unsigned long long)e.x << 32) | e.y;
          const uint32_t same = __match_any_sync(0xffffffffu, slot);
          if (has_slot && (same & lt_mask)) ok = false;
        }
        const uint32_t bad = ~__ballot_sync(0xffffffffu, ok) & act_mask;
        const uint32_t n_ok = bad ? (uint32_t)(__ffs(bad) - 1) : g;
        // ---- commit the clean prefix -----------------------------------------------
        if (lane < n_ok) {
          if (f) {
            a.res[ds.x] = stream_fail_res(f);
          } else {
            atomicMax(&run_s[e.x], e.y + 1);  // several lanes may take consecutive slots of one servant
            a.res[ds.x] = sv_begin + e.x;
            if (one_class) {
              if (lane == n_ok - 1) sh.front[c] += win_pos + 1;  // everything up to my entry is taken now
            } else {
              const uint32_t mine = peers & ((n_ok == 32) ? 0xffffffffu : ((1u << n_ok) - 1));
              if (rank == 0) sh.front[c] += __popc(mine);  // they took front .. front + count - 1
            }
          }
        }
        __syncwarp();
        at += n_ok;
        ++st_steps; st_lanes += n_ok;
        if (n_ok == g) continue;
        if (n_ok < (one_class ? 1u : 6u)) cooldown = 48;  // not worth it right now
      } else {
        --cooldown;
      }

      // ---- the first request that did not fit the pattern: exact walk ----------------
      const uint4 d1 = dl[at];
      ++at;
      ++st_walks;
      const uint32_t q = d1.x, c1 = d1.y;
      uint32_t selfinfo = d1.z;
      const uint8_t f1 = sh.fail[c1];
      if (f1) {
        if (lane == 0) a.res[q] = stream_fail_res(f1);
        continue;
      }
      // several servants on the requestor's IP: "self" is the first of them that is
      // eligible for this class and free right now (find_if over the free list, cc:372-375)
      if (selfinfo != kNone && (selfinfo & 0x80000000u)) {
        const uint32_t ip = selfinfo & 0x7FFFFFFFu;
        const uint32_t env = a.ct.cls_env[c1], mv = a.ct.cls_mv[c1];
        uint32_t best = kNone;
        for (uint32_t u0 = a.t.ip_off[ip], ue = a.t.ip_off[ip + 1]; u0 < ue && best == kNone; u0 += 32) {
          const uint32_t u = u0 + lane;
          uint32_t cand = kNone;
          if (u < ue) {
            const uint32_t p = a.t.ip_sv[u];
            if (a.t.sv_comp[p] == comp) {
              const uint32_t l = a.t.sv_local[p];
              if (a.sv.max_tasks[p] != 0 && (uint32_t)a.sv.version[p] >= mv && run_s[l] < lim_s[l] &&
                  servant_has_env(a.t, p, env)) {
                cand = l;
              }
            }
          }
          best = __reduce_min_sync(0xffffffffu, cand);  // CSR rows are in ascending position order
        }
        selfinfo = best;
      }
      const uint32_t selfl = selfinfo;
      const uint32_t end = sh.end[c1];
      uint32_t base = sh.front[c1];
      uint32_t new_front = base;
      bool front_open = true;
      uint32_t self_slot = kNone;  // the own servant's head slot, if the walk passed it
      uint32_t win = kNone;
      while (base < end) {
        ++st_windows;
        const uint32_t idx = base + lane;
        const bool valid = idx < end;
        uint2 w = make_uint2(0, 0);
        if (valid) w = a.list[idx];
        const bool taken = valid && w.y < run_s[w.x];
        const bool isself = valid && !taken && w.x == selfl;
        const bool avail = valid && !taken && !isself;
        const uint32_t bT = __ballot_sync(0xffffffffu, taken);
        const uint32_t bS = __ballot_sync(0xffffffffu, isself);
        const uint32_t bA = __ballot_sync(0xffffffffu, avail);
        if (front_open) {  // the front only ever moves over a contiguous run of taken slots
          const uint32_t lead = (bT == 0xffffffffu) ? 32u : (uint32_t)(__ffs(~bT) - 1);
          new_front += lead;
          if (lead < 32) front_open = false;
        }
        if (self_slot == kNone && bS) self_slot = selfl;
        if (bA) {
          const uint32_t wl = __ffs(bA) - 1;
          win = __shfl_sync(0xffffffffu, w.x, wl);
          if (base + wl == new_front) ++new_front;  // granted the front entry itself: it is taken now
          break;
        }
        base += 32;
      }
      if (win == kNone && self_slot != kNone) win = self_slot;  // last resort (cc:394-396)
      __syncwarp();
      if (lane == 0) {
        sh.front[c1] = new_front;
        if (win != kNone) {
          run_s[win] += 1;
          a.res[q] = sv_begin + win;
        } else {
          a.res[q] = kResTimeout;  // the class has eligible servants but none is free (cc:116-118)
          sh.fail[c1] = 1;         // ... and within this batch none will become free again
        }
      }
      __syncwarp();
    }
    if (t + 2 < n_tiles) bar_arrive(kBarFree0 + buf, nall);
  }

  if (lane == 0 && a.counters) {
    atomicAdd(&a.counters->pad[2], st_walks); atomicAdd(&a.counters->pad[3], st_windows);
  }
  // (++running_tasks / ++ever_assigned_tasks, cc:123-124, are applied per grant by k_final_write)
}

}  // namespace yd
