// parallel.cuh -- the data-parallel assignment path of the slot-stream solver.
//
// If every request that can reach a component belongs to ONE class (one digest,
// one min_version) and none of them comes from a machine that is itself a servant
// of that component, the sequential fold of task_dispatcher.cc:93-140 collapses:
// all requests see the same sorted slot list, nobody skips anything, so the j-th
// request of the class (FIFO order) takes the j-th slot of the list and requests
// beyond the list's end time out.  That is a per-class exclusive prefix count
// (the FIFO rank) followed by one gather -- no dependency between decisions.
//
//   (k_cls_finalize marks such components, comp_mode = 1; the sequential solver
//    in solve_stream.cuh skips them)
//   k_rank_count   per 1024-request tile: class of each request, its rank among the
//                  tile's requests of the same class (warp __match_any_sync + a
//                  32 x 256 shared-memory count table), per-(class, tile) totals
//   k_rank_assign  rank = scanned (class, tile) base + in-tile rank;
//                  grant list[rank] or Timeout / EnvironmentNotFound
#pragma once
#include "classes.cuh"

namespace yd {

constexpr int kRankTile = 1024;

// The FIFO rank of this thread's request (class `cls`, or kNone) among the requests of its class in tile `tile` (a block
// of 1024 threads, thread = position in the tile), and the tile's per-class totals: every (class, tile) cell of tile_cnt
// below cls_bound is written.
__device__ __forceinline__ uint32_t rank_in_tile(uint32_t tile, uint32_t cls, const ClassTable& ct, uint32_t n_tiles,
                                                 uint32_t* __restrict__ tile_cnt) {
  __shared__ uint16_t wc[32][kMaxClasses];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t i = tid; i < 32 * kMaxClasses / 2; i += kRankTile) reinterpret_cast<uint32_t*>(&wc[0][0])[i] = 0;
  __syncthreads();
  const uint32_t peers = __match_any_sync(0xffffffffu, cls);
  const uint32_t wrank = __popc(peers & ((1u << lane) - 1));
  if (cls != kNone && wrank == 0) wc[warp][cls] = (uint16_t)__popc(peers);
  __syncthreads();
  // exclusive prefix over the 32 warps, per class; tile total to HBM
  if (tid < ct.cls_bound) {
    uint32_t run = 0;
#pragma unroll 4
    for (int w = 0; w < 32; ++w) {
      const uint32_t c = wc[w][tid];
      wc[w][tid] = (uint16_t)run;
      run += c;
    }
    tile_cnt[tid * n_tiles + tile] = run;
  }
  if (tile == 0 && tid == 0) tile_cnt[ct.cls_bound * n_tiles] = 0;  // the scan's end cell
  __syncthreads();
  const uint32_t rank = cls != kNone ? (uint32_t)wc[warp][cls] + wrank : 0u;
  __syncthreads();  // (wc is reused when a block handles several tiles)
  return rank;
}

// One tile of 1024 requests (a block of 1024 threads).  Every (class, tile) cell of tile_cnt below cls_bound is written,
// so tiles beyond the end of the queue must be run too (their cells are zero).
__device__ __forceinline__ void rank_count_tile(uint32_t tile, const ReqView& reqs, uint32_t n,
                                                const TopoView& t, const ClassTable& ct,
                                                const uint32_t* __restrict__ comp_mode, uint32_t n_tiles,
                                                uint32_t* __restrict__ rcls, uint32_t* __restrict__ rrank,
                                                uint32_t* __restrict__ rself, uint32_t* __restrict__ tile_cnt) {
  const uint32_t q = tile * kRankTile + threadIdx.x;
  uint32_t cls = kNone, self = kNone;
  if (q < n) {
    uint32_t env, mv;
    reqs.head(q, env, mv);
    if (env < t.n_envs) {
      const uint32_t comp = t.env_comp[env];
      if (comp != kNone && comp_mode[comp] != 0) {  // data-parallel or merge: both need FIFO ranks
        const uint32_t slot = cls_find(ct.keys, ((unsigned long long)env << 32) | mv);
        if (slot != kNone) cls = ct.slot_cls[slot];
        if (cls != kNone && comp_mode[comp] == 2 && (ct.comp_flags[comp] & 1u)) {
          self = self_servant(t, reqs.ip(q), comp);
        }
      }
    }
  }
  const uint32_t rank = rank_in_tile(tile, cls, ct, n_tiles, tile_cnt);
  if (q < n) {
    rcls[q] = cls;
    rrank[q] = rank;
    rself[q] = self;
  }
}

__global__ void __launch_bounds__(kRankTile) k_rank_count(const yd_task_req* __restrict__ reqs,
                                                          const DynParams* __restrict__ dp, TopoView t, ClassTable ct,
                                                          const uint32_t* __restrict__ comp_mode, uint32_t n_tiles,
                                                          uint32_t* __restrict__ rcls,   // [n] class or kNone
                                                          uint32_t* __restrict__ rrank,  // [n] rank inside the tile
                                                          uint32_t* __restrict__ rself,  // [n] own servant (merge solver)
                                                          uint32_t* __restrict__ tile_cnt /* [kMaxClasses][n_tiles] */) {
  rank_count_tile(blockIdx.x, ReqView{reqs, nullptr}, dp->n, t, ct, comp_mode, n_tiles, rcls, rrank, rself, tile_cnt);
}

// Per-class layout of the merge solver's request records (RqLayout) for the range-sharded queue.  (One GPU: class
// c's records are its whole FIFO list, stored where the rank scan put it -- RqLayout derives that itself and this
// kernel is not launched.)  Called twice: first (`lcnt_all` == null) it only reports this rank's per-class
// request counts for the exchange; then (`lcnt_all` = every
// rank's per-class request counts, rank-major, cls_bound words per rank): this rank's requests of class
// c follow those of the lower ranks, and only the head of the class list that slots can reach is kept --
// one record per slot of the class's list plus a margin for requests passed over by their own servant
// (a request beyond it makes the merge solver hand the batch back, solve_merge.cuh).
constexpr uint32_t kRqMargin = 1024;

__global__ void __launch_bounds__(256) k_rq_layout(ClassTable ct, const uint32_t* __restrict__ comp_mode,
                                                   const uint32_t* __restrict__ rank_off, uint32_t n_rank_tiles,
                                                   const uint32_t* __restrict__ list_off, uint32_t n_list_tiles,
                                                   const uint32_t* __restrict__ lcnt_all, uint32_t rank, uint32_t world,
                                                   uint32_t* __restrict__ lcnt_out, RqLayout L) {
  __shared__ uint32_t s_win[kMaxClasses];
  const uint32_t ncls = min(ct.meta[0], ct.cls_bound);
  for (uint32_t c = threadIdx.x; c < ncls; c += blockDim.x) {
    const uint32_t mine = rank_off[(c + 1) * n_rank_tiles] - rank_off[c * n_rank_tiles];
    if (lcnt_out) lcnt_out[c] = mine;  // (sharded: what this rank contributes to the next exchange)
    if (lcnt_all) {
      uint32_t before = 0, all = 0;
      for (uint32_t g = 0; g < world; ++g) {
        const uint32_t v = lcnt_all[g * ct.cls_bound + c];
        if (g < rank) before += v;
        all += v;
      }
      const uint32_t len = list_off[(c + 1) * n_list_tiles] - list_off[c * n_list_tiles];
      L.goff[c] = before; L.gn[c] = all;
      s_win[c] = comp_mode[ct.cls_comp[c]] == 2 ? min(all, len + kRqMargin) : 0u;  // only the merge solver reads records
      L.win[c] = s_win[c];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    if (lcnt_all) {
      for (uint32_t c = 0; c < ncls; ++c) { L.base[c] = run; run += s_win[c]; }
    }
    *L.total = run;
  }
}

// tile_off = exclusive scan of tile_cnt over (class-major, tile-minor).
// The verdict of request q as far as it is known before the coupled solvers run: false = not ours (the sequential
// solver -- or nobody -- answers it; res[q] keeps kResEnvNotFound), else `out` = what goes into res[q].  Requests of
// merge-mode components also publish their FIFO record.
__device__ __forceinline__ bool rank_assign_one(uint32_t q, uint32_t n_tiles, const TopoView& t, const ClassTable& ct,
                                                const uint32_t* __restrict__ rcls, const uint32_t* __restrict__ rrank,
                                                const uint32_t* __restrict__ rself, const uint32_t* __restrict__ tile_off,
                                                const uint32_t* __restrict__ list_off, uint32_t n_list_tiles,
                                                const uint2* __restrict__ list, const uint32_t* __restrict__ comp_mode,
                                                uint2* __restrict__ rq, const RqLayout& L, uint32_t& out) {
  const uint32_t c = rcls[q];
  if (c == kNone) return false;  // not ours: the sequential solver (or nobody) answers it
  if (ct.cls_nelig[c] == 0) { out = kResEnvNotFound; return true; }  // cc:105-108
  // FIFO rank inside the class, over the whole queue (lower ranks' requests come first)
  const uint32_t rank = L.Goff(c) + tile_off[c * n_tiles + q / kRankTile] - tile_off[c * n_tiles] + rrank[q];
  if (comp_mode[ct.cls_comp[c]] == 2) {
    // merge solver: publish the class's FIFO request list (class c owns rq[tile_off[c][0] ...)) as
    // (request, its own servant in the component or kNone);
    // the verdict stays Timeout unless a slot picks this request (solve_merge.cuh)
    if (rank < L.Win(c)) rq[L.Base(c) + rank] = make_uint2(L.q_base + q, rself[q]);
    out = kResTimeout;
    return true;
  }
  const uint32_t lb = list_off[c * n_list_tiles], le = list_off[(c + 1) * n_list_tiles];
  if (rank >= le - lb) { out = kResTimeout; return true; }  // cc:116-118
  const uint2 e = list[lb + rank];  // (servant local index, running_tasks value of the slot)
  out = t.comp_sv_off[ct.cls_comp[c]] + e.x;  // (++running_tasks, ++ever_assigned_tasks happen in k_final_write)
  return true;
}

__global__ void __launch_bounds__(256) k_rank_assign(const DynParams* __restrict__ dp, uint32_t n_tiles, TopoView t,
                                                     ClassTable ct,
                                                     const uint32_t* __restrict__ rcls,
                                                     const uint32_t* __restrict__ rrank,
                                                     const uint32_t* __restrict__ rself,
                                                     const uint32_t* __restrict__ tile_off,
                                                     const uint32_t* __restrict__ list_off, uint32_t n_list_tiles,
                                                     const uint2* __restrict__ list, ServantArrays sv,
                                                     const uint32_t* __restrict__ comp_mode,
                                                     uint2* __restrict__ rq, uint32_t* __restrict__ res, RqLayout L) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= dp->n) return;
  // Overflow flagged by the class table or the list builder: the host reruns this batch (bigger
  // class bound or the row-scan solver), so nothing may be decided -- or counted -- now.
  if (ct.meta[1]) return;
  uint32_t v;
  if (rank_assign_one(q, n_tiles, t, ct, rcls, rrank, rself, tile_off, list_off, n_list_tiles, list, comp_mode, rq, L, v)) res[q] = v;
}

}  // namespace yd
