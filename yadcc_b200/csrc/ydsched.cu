// ydsched.cu -- host side of the H100-native scheduler hot path and its C ABI
// (include/ydsched.h).  This translation unit owns:
//
//   * the servant registry mirror (strings, digests, leases) -- the part of
//     TaskDispatcher that is string handling, not arithmetic
//     (KeepServantAlive cc:190-220, the expiry decision of OnExpirationTimer
//     cc:503-516, RunningTaskBookkeeper);
//   * the topology builder: digest<->servant components, per-component digest
//     membership bit tables, requestor-ip -> servant CSR;
//   * the launch sequences for the kernels in slots.cuh / solve_rowscan.cuh /
//     tasks.cuh.  All arithmetic of the hot path (eligibility, capacity,
//     utilisation, pick, task ids, leases, sweeps) runs on the GPU.
//
// There is no CPU fallback: yd_create fails without an sm_90 device.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <type_traits>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "slots.cuh"
#include "radix.cuh"
#include "solve_rowscan.cuh"
#include "solve_stream.cuh"
#include "parallel.cuh"
#include "solve_merge.cuh"
#include "bloom.cuh"
#include "running_index.cuh"
#include "tasks.cuh"
#include "tiny.cuh"
#include "fused.cuh"
#include "filter.cuh"
#include "rpcs.cuh"
#include "blake3.cuh"
#include "state.cuh"
#include "ydstate_codec.inc"
#include "ydkeys.h"
#include "ydshard.h"
#include "ydruns.h"
#include "ydrpcs_packed.h"
#include "ydsched_keys_impl.inc"

namespace {

using yd::Counters;
using yd::kNone;

// ---- small helpers ---------------------------------------------------------

// Bumped whenever any device buffer moves: captured graphs hold raw pointers.  (Atomic: several handles may run
// in threads of one process, e.g. the ranks of a range-sharded scheduler.)
static std::atomic<unsigned long long> g_buf_generation{0};

struct DevBuf {  // grow-only device allocation
  void* p = nullptr;
  size_t cap = 0;
  template <class T> T* as() const { return static_cast<T*>(p); }
  void ensure(size_t bytes, bool keep = false, cudaStream_t st = nullptr) {
    if (bytes <= cap) return;
    size_t ncap = std::max(bytes, cap * 2);
    ncap = (ncap + 255) & ~size_t(255);
    void* np = nullptr;
    YD_CUDA_CHECK(cudaMalloc(&np, ncap));
    if (keep && p && cap) YD_CUDA_CHECK(cudaMemcpyAsync(np, p, cap, cudaMemcpyDeviceToDevice, st));
    if (p) {
      YD_CUDA_CHECK(cudaStreamSynchronize(st));
      YD_CUDA_CHECK(cudaFree(p));
    }
    p = np;
    cap = ncap;
    ++g_buf_generation;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    ++g_buf_generation;
  }
};

struct PinBuf {  // grow-only pinned host staging
  void* p = nullptr;
  size_t cap = 0;
  template <class T> T* as() const { return static_cast<T*>(p); }
  void ensure(size_t bytes) {
    if (bytes <= cap) return;
    size_t ncap = std::max(bytes, cap * 2);
    if (p) YD_CUDA_CHECK(cudaFreeHost(p));
    YD_CUDA_CHECK(cudaHostAlloc(&p, ncap, cudaHostAllocDefault));
    cap = ncap;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

// yadcc::TryParseSize, yadcc/common/parse_size.cc:25-45.
bool ParseSize(const char* text, uint64_t* out) {
  if (!text) return false;
  size_t len = strlen(text);
  if (len == 0) return false;
  uint64_t scale = 1;
  switch (text[len - 1]) {
    case 'G': scale = 1ull << 30; --len; break;
    case 'M': scale = 1ull << 20; --len; break;
    case 'K': scale = 1ull << 10; --len; break;
    case 'B': --len; break;
    default: break;
  }
  if (len == 0) return false;
  uint64_t v = 0;
  for (size_t i = 0; i != len; ++i) {
    if (text[i] < '0' || text[i] > '9') return false;
    uint64_t nv = v * 10 + uint64_t(text[i] - '0');
    if (nv / 10 != v) return false;
    v = nv;
  }
  *out = v * scale;
  return true;
}

struct ServantHost {  // ServantPersonality + ServantDesc lease fields (h:80-116,184-193)
  int32_t version = 0;
  std::string observed, reported;
  std::vector<uint32_t> envs;  // interned digest ids, heartbeat order (duplicates kept)
  uint32_t nproc = 0, load = 0, max_tasks = 0;
  uint64_t total_mem = 0, avail_mem = 0;
  int32_t priority = 0, reason = 0;
  int64_t discovered_at = 0, expires_at = 0;
};

struct RunningRec {
  uint64_t servant_task_id, task_grant_id;
  std::string servant_location, task_digest;
  // Index of the task in the heartbeat that reported it.  A rank of a range-sharded queue keeps only the reported tasks
  // whose lease it holds; the ranks' groups merged by this index are the single scheduler's (yd_shard_export_state).
  uint32_t report_pos = 0;
};

// The sequence of a slot-stream solve (EnqueueSolve); the YDSCHED_DEBUG line prints the number.
enum SolveVariant : uint32_t {
  kPipeline = 0,   // the kernel-by-kernel pipeline
  kFused = 1,      // fused front (fused.cuh) + coupled solvers + final
  kSolo = 2,       // the fused front alone: it writes the grants too
  kSoloClean = 3,  // the same on a clean scratch (no memset nodes)
  kSoloSpec = 4,   // solo and speculative on the kept class table (no memsets)
};
constexpr bool IsSolo(SolveVariant v) { return v == kSolo || v == kSoloClean || v == kSoloSpec; }

// One attempt of a solve.  A stand-down escalates the merge rounds or the solver here, never in the configured values.
struct SolvePlan {
  SolveVariant variant;
  uint32_t solver;        // 1 row scan, 2 slot streams
  uint32_t merge_rounds;  // (a graph key: a settled merge needs fewer)
  uint32_t force_stream;  // ClassTable::force_stream
  // Flag 3 (the merge did not settle): eight times the rounds, at most as many as the merge has chunks (+ 2).
  void MoreMergeRounds(uint32_t max_chunks) { merge_rounds = std::min(merge_rounds * 8, max_chunks + 2); }
};

// The solo kernel re-initialises the scratch it dirtied (class-table keys, zeroed region) before it ends; while this
// signature matches the current buffers and layout the next solo solve needs no memset nodes either.
struct CleanSig { unsigned long long gen = ~0ull; size_t z_cls_off = 0, z_bytes = 0, res_words = 0; const void* zero = nullptr; const void* res = nullptr;
  bool operator==(const CleanSig& o) const { return gen == o.gen && z_cls_off == o.z_cls_off && z_bytes == o.z_bytes && res_words == o.res_words && zero == o.zero && res == o.res; } };
// A kept class table is valid for the buffers, the topology and the class bound it was built with.
struct KeptSig { CleanSig clean; unsigned long long topo_gen = 0; uint32_t cls_bound = 0;
  bool operator==(const KeptSig& o) const { return clean == o.clean && topo_gen == o.topo_gen && cls_bound == o.cls_bound; } };

// What one solve leaves the next about the fused solo kernel (fused.cuh).  A solo solve that finds the class set of the
// previous one keeps its class table, and the next solo solve runs the speculative variant on it.  kept_fp = the
// class-set fingerprint of the last non-speculative solo solve (0: none -- nothing to compare with, as after a
// speculative solve missed): speculation resumes only after two such solves in a row agree.
struct SoloTables {
  bool hint = true;  // the last batch consisted of data-parallel components only
  CleanSig clean;
  bool clean_valid = false;
  KeptSig kept;
  bool kept_valid = false;
  unsigned long long kept_fp = 0;

  // The variant of an attempt; `fused`: the fused kernel may take the batch, `now`: the scratch, topology and class
  // bound it would run on, `spec_ok`: the batch fits the speculative variant.  Whatever runs dirties the scratch, and
  // anything but the speculative variant rebuilds or clears the kept table.
  SolveVariant Choose(bool fused, const KeptSig& now, bool spec_ok) {
    const SolveVariant v = !fused ? kPipeline : !hint ? kFused
                         : kept_valid && kept == now && spec_ok ? kSoloSpec
                         : clean_valid && clean == now.clean ? kSoloClean : kSolo;
    clean_valid = false;
    if (v != kSoloSpec) kept_valid = false;
    return v;
  }
  // After an attempt of `v` on `now`: `meta` = the class table's meta words (meta[1]: the flag), `fp` = the solo
  // kernel's class-set fingerprint.
  void Take(SolveVariant v, const uint32_t* meta, const KeptSig& now, unsigned long long fp) {
    if (meta[1] == yd::kFlagSpecMiss) {
      // the kernel left the scratch clean; the replay builds the table again
      kept_valid = false;
      kept_fp = 0;
      clean = now.clean;
      clean_valid = true;
    } else if (meta[1] == 4) {  // a component the solo kernel cannot decide: the general sequence, now and next time
      hint = false;
    } else if (meta[1] == 0 && v == kFused) {
      hint = meta[4] == 0;  // back to one launch when nothing is coupled any more
    } else if (meta[1] == 0 && (v == kSolo || v == kSoloClean)) {
      // the kernel's last block has kept the class table (same class set as the previous such solve) or cleared it,
      // and re-initialised the rest of the scratch.  (A completed speculative solve leaves the kept table valid.)
      if (fp == kept_fp) {
        kept = now;
        kept_valid = true;
      } else {
        clean = now.clean;
        clean_valid = true;
      }
      kept_fp = fp;
    }
  }
  // Another sequence (the sharded solve) dirtied the scratch and overwrote the class table.
  void Drop() { clean_valid = kept_valid = false; }
};

}  // namespace

struct yd_shard_ctx;  // range-sharded queue over several GPUs (shard_host.inc)

struct yd_sched {
  int device = 0;
  yd_shard_ctx* shard = nullptr;
  cudaStream_t st = nullptr;
  uint64_t min_mem = 0;
  uint32_t solver_pref = 0;

  // interning
  std::vector<std::string> envs, ips;
  std::unordered_map<std::string, uint32_t> env_ids, ip_ids;

  // registry mirror
  std::vector<ServantHost> sv;
  std::unordered_map<std::string, uint32_t> loc2pos;
  bool topo_dirty = true, facts_dirty = true;
  // The sorted slot order depends on the heartbeat facts only (key(s, r) is static, slots.cuh): it is built when
  // a capacity fact, a priority or the servant set changes and kept across solves; a solve only filters out the
  // slots servants have filled meanwhile.  (Above kStaticSlotLimit slots the table is rebuilt per solve, clamped
  // to the batch size.)
  bool order_dirty = true, order_static = false;
  size_t order_slot_b = 0;
  unsigned long long order_rebuilds = 0;

  // device servant arrays; state (run/ever) is valid for positions < S_dev
  DevBuf d_nproc, d_load, d_maxt, d_flags, d_ver, d_run, d_ever;
  DevBuf d_run_tmp, d_ever_tmp, d_remap;
  DevBuf d_dec, d_dec_tmp;  // range-sharded handles: running_tasks decrements not yet handed to the other ranks
  uint32_t S_dev = 0;
  PinBuf h_facts;

  // topology on device
  DevBuf d_env_comp, d_env_local, d_comp_sv_off, d_comp_sv, d_comp_mask_off, d_comp_nwarps, d_envmask,
      d_sv_comp, d_sv_local, d_ip_off, d_ip_sv, d_ip_comp_mask;
  DevBuf d_kept_env, d_kept_sv;  // the kept class table per digest / per servant (fused.cuh)
  uint32_t n_comps = 0, n_envs_dev = 0, n_ips_dev = 0, max_warps = 1, max_comp_servants = 0;
  bool wide = false;
  PinBuf h_topo;

  // slot-stream solver state
  DevBuf d_sv_env_off, d_sv_envs, d_comp_mode, d_sv_emask, d_slot_rec, d_slot_spos;
  bool emask_ok = false;  // every component holds <= 64 digests: d_sv_emask is valid
  DevBuf d_slot_owner, d_sort_k[2], d_sort_v[2];
  // one zero-filled scratch region per solve: radix histograms (one per pass), the class
  // table's u32 arrays, the per-(class, tile) list counts -- a single memset node
  DevBuf d_zero;
  size_t z_hist_off[10] = {}, z_cls_off = 0, z_listcnt_off = 0, z_bytes = 0;
  uint32_t sort_nb = 0;
  cudaStream_t st2 = nullptr, st_copy = nullptr;  // class/rank branch; request upload
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_h2d = nullptr, ev_fin = nullptr;
  uint32_t cls_bound = 16;  // classes the per-class grids are sized for; grows on demand (<= yd::kMaxClasses)
  DevBuf d_list, d_list_bal, d_rcls, d_rrank, d_rank_cnt, d_rq, d_rself;
  DevBuf d_members;  // the fused solo solve's per-tile member lists (classes.cuh: list_member_index)
  // merge solver (solve_merge.cuh): per-slot verdicts and the chunk boundary states
  DevBuf d_slot_pick, d_mst_in, d_mst_out, d_stream_scratch;
  size_t z_merge_off = 0, z_layout_off = 0, z_final_off = 0, z_scan_off = 0;
  uint32_t merge_max_chunks = 0, merge_grid = 0, merge_grid_kcap = 0;
  // configured at yd_create; a solve starts from these and escalates in its own SolvePlan
  uint32_t cfg_merge_chunk = 0;    // YDSCHED_MERGE_CHUNK (0: by batch size, MergeChunk)
  uint32_t cfg_merge_rounds = 16;  // YDSCHED_MERGE_ROUNDS
  uint32_t cfg_force_stream = 0;   // yd_config.reserved bit 1 / YDSCHED_FORCE_STREAM: no merge solver for self-requests
  bool debug_env = false, tiny_ok = true;
  bool stream_attr_set = false;
  // fused front kernel (fused.cuh): one persistent launch for the class / rank / list phases and -- `solo` -- the grants
  bool fused_cfg = true;       // yd_config.reserved bit 3 / YDSCHED_NO_FUSED switch it off
  uint32_t fused_grid = 0;    // blocks of the fused kernel: one per SM
  uint32_t fused_max_nb = 262144;  // largest batch size class that takes it (YDSCHED_FUSED_MAX_N)
  size_t z_fbar_off = 0;
  DevBuf d_reqs16, d_out8;     // packed upload / download (yd_task_req16, yd_grant8)
  yd::FusedHostIO* h_fio = nullptr;  // mapped pinned record: the solo kernel's result (no copy after its launch)
  yd::FusedHostIO* d_fio = nullptr;  // its device-side address
  yd::FusedScalars fsc{};            // the call's scalars: kernel parameters of a solo launch ...
  PinBuf h_fsc;                      // ... or (graphed general sequence) copied into d_fsc by the graph's first node
  DevBuf d_fsc;
  SoloTables solo;
  bool fused_prof = false;    // YDSCHED_FUSED_PROF: phase stamps of the fused kernel, printed after every solve
  DevBuf d_fused_prof;
  size_t res_words = 0;  // u32 words of res[] in d_res (the class-table keys follow)
  size_t staged_n = 0;   // requests placed in d_reqs by yd_stage_requests

  // lease ring
  DevBuf d_t_exp, d_t_srv, d_t_flags;
  uint64_t ring_cap = 0;
  uint64_t lo = 0, next_id = 0;
  uint32_t id_stride = 1, id_offset = 0;
  uint64_t zombies_ub = 0;

  // per-solve buffers
  DevBuf d_reqs, d_res, d_out, d_blk, d_row_off, d_row_len, d_codes, d_ids, d_ok;
  DevBuf d_counters;
  PinBuf h_counters, h_small;

  // RunningTaskBookkeeper (running_task_bookkeeper.h:41-42): same container, same
  // operation sequence as the reference, hence the same iteration order.
  std::unordered_map<std::string, std::vector<RunningRec>> running;
  std::vector<RunningRec> running_cache;
  std::vector<const char*> personality_envs;  // backing store for yd_get_servant_personality

  // captured solve graphs, keyed by size class
  struct GraphKey {
    uint32_t Nb = 0, S = 0, n_comps = 0, max_comp = 0, cls_bound = 0, solver = 0, wide = 0, merge_rounds = 0, force_stream = 0,
             order_static = 0, packed = 0;
    SolveVariant variant = kPipeline;
    size_t slot_b = 0;
    unsigned long long gen = 0, topo_gen = 0;  // buffer reallocations; topology rebuilds (n_envs, n_ips, ... are baked in)
    uint64_t ring_cap = 0;
    bool operator==(const GraphKey& o) const {
      return Nb == o.Nb && S == o.S && n_comps == o.n_comps && max_comp == o.max_comp && cls_bound == o.cls_bound &&
             merge_rounds == o.merge_rounds && force_stream == o.force_stream && order_static == o.order_static &&
             solver == o.solver && wide == o.wide && slot_b == o.slot_b && gen == o.gen && topo_gen == o.topo_gen &&
             ring_cap == o.ring_cap && variant == o.variant && packed == o.packed;
    }
  };
  struct GraphEntry {
    GraphKey key;
    cudaGraphExec_t exec = nullptr;
    uint32_t launches = 0;
  };
  bool host_prof = false;      // YDSCHED_HOST_PROF: host-side timestamps of a solve, printed
  std::vector<GraphEntry> graphs;
  unsigned long long topo_gen = 0;
  bool use_graphs = true;
  DevBuf d_dyn;
  PinBuf h_dyn, h_meta;

  // compilation-cache bloom pre-filter
  DevBuf d_bloom, d_bloom_keys, d_bloom_out;
  uint64_t bloom_bits = 0;
  uint32_t bloom_hashes = 0;

  // in-flight task index (running_index.cuh)
  std::vector<RunningRec> rt_snapshot;
  DevBuf d_rt_bytes, d_rt_off, d_rt_len, d_rt_ids, d_rt_slots, d_rt_keys, d_rt_out;
  DevBuf d_freqs, d_fverdict, d_ftile;  // pre-filtered solve (filter.cuh): the unfiltered queue, verdicts, tile counts
  // a window of RPCs decided on the device (rpcs.cuh): the records, where each RPC's decisions start, its grant counts
  // (scanned: first_grant), the results, the reported grants
  DevBuf d_rpcs, d_rpc_off, d_rpc_ng, d_rpc_res, d_rpc_out;
  PinBuf h_fcount;
  cudaEvent_t ev_f[2] = {};
  // the env table on the device (blake3.cuh): digest e = env_bytes[env_off[e] .. env_off[e + 1]) for e < env_dev_n,
  // appended from `envs` before a derivation reads it.  Allocated stream-ordered, outside the grow-only buffers.
  unsigned char* d_env_bytes = nullptr;
  uint32_t* d_env_off = nullptr;
  size_t env_dev_n = 0, env_dev_bytes = 0, env_cap_n = 0, env_cap_bytes = 0;
  uint32_t rt_mask = 0;
  size_t rt_distinct = 0;

  cudaEvent_t ev[6] = {};
  yd_solve_stats stats{};
  bool have_stats = false;
  int stats_times_pending = 0;  // 1: events of an eager general solve, 2: of a graphed or solo one, not yet turned into milliseconds
  size_t static_bound_cache = 0;  // the sum over the servants of min(nproc, max_tasks) + 1 (SyncFacts): the kept slot table's bound

  yd::ServantArrays arrays() const {
    return yd::ServantArrays{d_nproc.as<uint32_t>(), d_load.as<uint32_t>(), d_maxt.as<uint32_t>(),
                             d_flags.as<uint32_t>(), d_ver.as<int32_t>(), d_run.as<uint32_t>(),
                             d_ever.as<unsigned long long>()};
  }
  yd::TaskRing ring() const {
    return yd::TaskRing{d_t_exp.as<long long>(), d_t_srv.as<uint32_t>(), d_t_flags.as<uint32_t>(),
                        ring_cap - 1, lo, next_id, id_stride, id_offset};
  }

  uint32_t InternEnv(const std::string& k) {
    auto it = env_ids.find(k);
    if (it != env_ids.end()) return it->second;
    uint32_t id = (uint32_t)envs.size();
    envs.push_back(k);
    env_ids.emplace(k, id);
    return id;
  }
  uint32_t InternIp(const std::string& k) {
    auto it = ip_ids.find(k);
    if (it != ip_ids.end()) return it->second;
    uint32_t id = (uint32_t)ips.size();
    ips.push_back(k);
    ip_ids.emplace(k, id);
    return id;
  }

  uint32_t FactFlags(const ServantHost& s) const {
    uint32_t f = 0;
    if (s.priority == YD_PRIORITY_DEDICATED) f |= yd::kFlagDedicated;
    if (s.total_mem != 0 && s.avail_mem < min_mem) f |= yd::kFlagLowMem;  // cc:286-292
    return f;
  }

  void EnsureRing(uint64_t need_ids);
  void SyncServantState();
  void SyncFacts();
  void SyncTopology();
  void FetchCounters();
};

// ---- device state maintenance ------------------------------------------------

// Extend run[] / ever[] with zeros for servants appended since the last sync
// (a new ServantDesc starts with running_tasks = 0, cc:208).
void yd_sched::SyncServantState() {
  uint32_t S = (uint32_t)sv.size();
  if (S <= S_dev) return;
  d_run.ensure(size_t(S) * 4, true, st);
  d_ever.ensure(size_t(S) * 8, true, st);
  YD_CUDA_CHECK(cudaMemsetAsync(d_run.as<uint32_t>() + S_dev, 0, size_t(S - S_dev) * 4, st));
  YD_CUDA_CHECK(cudaMemsetAsync(d_ever.as<unsigned long long>() + S_dev, 0, size_t(S - S_dev) * 8, st));
  if (shard) {
    d_dec.ensure(size_t(S) * 4, true, st);
    YD_CUDA_CHECK(cudaMemsetAsync(d_dec.as<uint32_t>() + S_dev, 0, size_t(S - S_dev) * 4, st));
  }
  S_dev = S;
}

void yd_sched::SyncFacts() {
  if (!facts_dirty) return;
  uint32_t S = (uint32_t)sv.size();
  if (S) {
    h_facts.ensure(size_t(S) * 20);
    uint32_t* h = h_facts.as<uint32_t>();
    uint32_t maxcap = 0;
    for (uint32_t i = 0; i != S; ++i) {
      const ServantHost& s = sv[i];
      h[i] = s.nproc;
      h[S + i] = s.load;
      h[2 * S + i] = s.max_tasks;
      h[3 * S + i] = FactFlags(s);
      h[4 * S + i] = (uint32_t)s.version;
      maxcap = std::max(maxcap, std::min(s.nproc, s.max_tasks));
    }
    static_bound_cache = 0;
    for (uint32_t i = 0; i != S; ++i) static_bound_cache += size_t(std::min(sv[i].nproc, sv[i].max_tasks)) + 1;
    if (wide != (maxcap > yd::kNarrowCapLimit)) order_dirty = true;
    wide = maxcap > yd::kNarrowCapLimit;
    d_nproc.ensure(size_t(S) * 4); d_load.ensure(size_t(S) * 4); d_maxt.ensure(size_t(S) * 4);
    d_flags.ensure(size_t(S) * 4); d_ver.ensure(size_t(S) * 4);
    YD_CUDA_CHECK(cudaMemcpyAsync(d_nproc.p, h, size_t(S) * 4, cudaMemcpyHostToDevice, st));
    YD_CUDA_CHECK(cudaMemcpyAsync(d_load.p, h + S, size_t(S) * 4, cudaMemcpyHostToDevice, st));
    YD_CUDA_CHECK(cudaMemcpyAsync(d_maxt.p, h + 2 * S, size_t(S) * 4, cudaMemcpyHostToDevice, st));
    YD_CUDA_CHECK(cudaMemcpyAsync(d_flags.p, h + 3 * S, size_t(S) * 4, cudaMemcpyHostToDevice, st));
    YD_CUDA_CHECK(cudaMemcpyAsync(d_ver.p, h + 4 * S, size_t(S) * 4, cudaMemcpyHostToDevice, st));
    // h_facts is reused by the next SyncFacts: make sure the DMA has read it.
    YD_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  facts_dirty = false;
}

// Components of the digest<->servant graph, digest membership bit tables and the
// requestor-ip CSR.  Runs only when the servant set or a digest list changed.
void yd_sched::SyncTopology() {
  if (!topo_dirty) return;
  const uint32_t S = (uint32_t)sv.size();
  const uint32_t E = (uint32_t)envs.size();
  // union-find over servants, joined through shared digests
  std::vector<uint32_t> parent(S);
  std::iota(parent.begin(), parent.end(), 0u);
  auto find = [&](uint32_t x) {
    while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; }
    return x;
  };
  std::vector<uint32_t> env_first(E, kNone);
  for (uint32_t i = 0; i != S; ++i) {
    for (uint32_t e : sv[i].envs) {
      if (env_first[e] == kNone) { env_first[e] = i; continue; }
      uint32_t a = find(env_first[e]), b = find(i);
      if (a != b) parent[std::max(a, b)] = std::min(a, b);
    }
  }
  std::vector<uint32_t> comp_of_root(S, kNone), sv_comp(S, kNone), sv_local(S, kNone);
  std::vector<std::vector<uint32_t>> comp_sv, comp_envs;
  for (uint32_t i = 0; i != S; ++i) {
    if (sv[i].envs.empty()) continue;  // can never be eligible
    uint32_t r = find(i);
    if (comp_of_root[r] == kNone) {
      comp_of_root[r] = (uint32_t)comp_sv.size();
      comp_sv.emplace_back();
      comp_envs.emplace_back();
    }
    uint32_t c = comp_of_root[r];
    sv_comp[i] = c;
    sv_local[i] = (uint32_t)comp_sv[c].size();
    comp_sv[c].push_back(i);
  }
  std::vector<uint32_t> env_comp(E, kNone), env_local(E, kNone);
  for (uint32_t i = 0; i != S; ++i) {
    for (uint32_t e : sv[i].envs) {
      if (env_comp[e] != kNone) continue;
      uint32_t c = sv_comp[i];
      env_comp[e] = c;
      env_local[e] = (uint32_t)comp_envs[c].size();
      comp_envs[c].push_back(e);
    }
  }
  const uint32_t C = (uint32_t)comp_sv.size();
  std::vector<uint32_t> sv_off(C + 1, 0), mask_off(C, 0), nwarps(C, 1), flat_sv;
  size_t mask_bytes = 0;
  max_warps = 1;
  for (uint32_t c = 0; c != C; ++c) {
    sv_off[c] = (uint32_t)flat_sv.size();
    flat_sv.insert(flat_sv.end(), comp_sv[c].begin(), comp_sv[c].end());
    uint32_t w = (uint32_t)((comp_sv[c].size() + 32 * yd::kK - 1) / (32 * yd::kK));
    nwarps[c] = std::max(1u, std::min(w, 32u));  // > 32 warps: only the slot-stream solver applies
    max_warps = std::max(max_warps, nwarps[c]);
    mask_off[c] = (uint32_t)mask_bytes;
    mask_bytes += size_t(comp_envs[c].size()) * nwarps[c] * 32;
  }
  sv_off[C] = (uint32_t)flat_sv.size();
  std::vector<uint8_t> envmask(std::max<size_t>(mask_bytes, 1), 0);
  for (uint32_t i = 0; i != S; ++i) {
    uint32_t c = sv_comp[i];
    if (c == kNone) continue;
    uint32_t l = sv_local[i], T = nwarps[c] * 32;
    if (l / yd::kK >= T) continue;  // component beyond the row-scan solver's 8192 servants: it never reads these masks
    for (uint32_t e : sv[i].envs) {
      envmask[mask_off[c] + size_t(env_local[e]) * T + l / yd::kK] |= uint8_t(1u << (l % yd::kK));
    }
  }
  // requestor-ip CSR: IsNetworkAddressEqual(ip_port, ip) (cc:66-69) holds iff `ip`
  // is a prefix of the observed location that ends right before a ':'.
  std::vector<std::vector<uint32_t>> by_ip(ips.size());
  for (uint32_t i = 0; i != S; ++i) {
    const std::string& loc = sv[i].observed;
    for (size_t k = 0; k < loc.size(); ++k) {
      if (loc[k] != ':') continue;
      uint32_t id = InternIp(loc.substr(0, k));
      if (id >= by_ip.size()) by_ip.resize(id + 1);
      by_ip[id].push_back(i);
    }
  }
  const uint32_t NI = (uint32_t)by_ip.size();
  std::vector<uint32_t> ip_off(NI + 1, 0), ip_sv;
  for (uint32_t k = 0; k != NI; ++k) {
    ip_off[k] = (uint32_t)ip_sv.size();
    ip_sv.insert(ip_sv.end(), by_ip[k].begin(), by_ip[k].end());
  }
  ip_off[NI] = (uint32_t)ip_sv.size();
  // the same per IP as one word: the components (< 64) with a servant on it (the speculative solve's self-request test)
  std::vector<unsigned long long> ip_comp_mask(std::max(NI, 1u), 0ull);
  for (uint32_t k = 0; k != NI; ++k) {
    for (uint32_t i : by_ip[k]) if (sv_comp[i] < 64) ip_comp_mask[k] |= 1ull << sv_comp[i];
  }

  auto up = [&](DevBuf& b, const void* src, size_t bytes) {
    b.ensure(std::max<size_t>(bytes, 4));
    if (bytes) YD_CUDA_CHECK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, st));
  };
  up(d_env_comp, env_comp.data(), size_t(E) * 4);
  up(d_env_local, env_local.data(), size_t(E) * 4);
  up(d_comp_sv_off, sv_off.data(), size_t(C + 1) * 4);
  up(d_comp_sv, flat_sv.data(), flat_sv.size() * 4);
  up(d_comp_mask_off, mask_off.data(), size_t(C) * 4);
  up(d_comp_nwarps, nwarps.data(), size_t(C) * 4);
  up(d_envmask, envmask.data(), envmask.size());
  up(d_sv_comp, sv_comp.data(), size_t(S) * 4);
  up(d_sv_local, sv_local.data(), size_t(S) * 4);
  up(d_ip_off, ip_off.data(), size_t(NI + 1) * 4);
  up(d_ip_sv, ip_sv.data(), ip_sv.size() * 4);
  up(d_ip_comp_mask, ip_comp_mask.data(), ip_comp_mask.size() * 8);
  d_kept_env.ensure(std::max<size_t>(size_t(E) * 16, 16));  // (both written by the solve that keeps a class table)
  d_kept_sv.ensure(std::max<size_t>(size_t(S) * 4, 4));
  // digest ids per servant (CSR) for class-eligibility tests on the device
  std::vector<uint32_t> env_off(S + 1, 0), env_flat;
  for (uint32_t i = 0; i != S; ++i) {
    env_off[i] = (uint32_t)env_flat.size();
    env_flat.insert(env_flat.end(), sv[i].envs.begin(), sv[i].envs.end());
  }
  env_off[S] = (uint32_t)env_flat.size();
  up(d_sv_env_off, env_off.data(), size_t(S + 1) * 4);
  up(d_sv_envs, env_flat.data(), env_flat.size() * 4);
  // digest membership as a 64-bit word per servant, when every component's digests fit
  emask_ok = true;
  for (uint32_t c = 0; c != C; ++c) emask_ok = emask_ok && comp_envs[c].size() <= 64;
  std::vector<unsigned long long> emask(std::max(S, 1u), 0ull);
  if (emask_ok) {
    for (uint32_t i = 0; i != S; ++i) for (uint32_t e : sv[i].envs) emask[i] |= 1ull << env_local[e];
  }
  up(d_sv_emask, emask.data(), emask.size() * 8);
  std::vector<uint32_t> comp_mode(std::max(C, 1u), 0);
  up(d_comp_mode, comp_mode.data(), comp_mode.size() * 4);
  max_comp_servants = 0;
  for (uint32_t c = 0; c != C; ++c) max_comp_servants = std::max<uint32_t>(max_comp_servants, (uint32_t)comp_sv[c].size());
  YD_CUDA_CHECK(cudaStreamSynchronize(st));  // sources are pageable temporaries
  n_comps = C;
  n_envs_dev = E;
  n_ips_dev = NI;
  topo_dirty = false;
  ++topo_gen;
}

void yd_sched::EnsureRing(uint64_t need_ids) {
  uint64_t need = (next_id - lo) + need_ids;
  if (ring_cap && need <= ring_cap) return;
  uint64_t ncap = ring_cap ? ring_cap : (1ull << 16);
  while (ncap < need * 2) ncap <<= 1;
  DevBuf ne, ns, nf;
  ne.ensure(ncap * 8); ns.ensure(ncap * 4); nf.ensure(ncap * 4);
  YD_CUDA_CHECK(cudaMemsetAsync(nf.p, 0, ncap * 4, st));
  if (ring_cap && next_id > lo) {
    yd::TaskRing nr{ne.as<long long>(), ns.as<uint32_t>(), nf.as<uint32_t>(), ncap - 1, lo, next_id, id_stride, id_offset};
    uint64_t cnt = next_id - lo;
    yd::k_ring_grow<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(ring(), nr);
    YD_CUDA_CHECK(cudaGetLastError());
  }
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  d_t_exp.release(); d_t_srv.release(); d_t_flags.release();
  d_t_exp = ne; d_t_srv = ns; d_t_flags = nf;
  ring_cap = ncap;
}

void yd_sched::FetchCounters() {
  YD_CUDA_CHECK(cudaMemcpyAsync(h_counters.p, d_counters.p, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
}

// ---- C ABI -------------------------------------------------------------------

extern "C" {

const char* yd_backend_name(void) { return "cuda-sm90a"; }

int yd_parse_size(const char* text, uint64_t* out_bytes) { return ParseSize(text, out_bytes) ? 1 : 0; }

yd_sched* yd_create(const yd_config* cfg) {
  if (!cfg || cfg->abi_version != YD_ABI_VERSION) return nullptr;
  uint64_t min_mem = 0;
  const char* mm = cfg->servant_min_memory_for_accepting_new_task;
  if (!ParseSize(mm ? mm : "10G", &min_mem)) return nullptr;  // cc:83-87
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev) {
    fprintf(stderr, "ydsched: no CUDA device %d (found %d); this backend has no CPU fallback\n",
            cfg->device, ndev);
    return nullptr;
  }
  cudaDeviceProp prop{};
  YD_CUDA_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 and nothing else
    fprintf(stderr, "ydsched: device %d is sm_%d%d; kernels are built for sm_90a only\n", cfg->device,
            prop.major, prop.minor);
    return nullptr;
  }
  YD_CUDA_CHECK(cudaSetDevice(cfg->device));
  auto* s = new yd_sched;
  s->device = cfg->device;
  s->min_mem = min_mem;
  s->solver_pref = cfg->solver;
  s->id_stride = cfg->id_stride ? cfg->id_stride : 1;
  s->id_offset = cfg->id_stride ? cfg->id_offset : 0;
  s->use_graphs = !(cfg->reserved & 1u) && !getenv("YDSCHED_NO_GRAPH");
  s->cfg_force_stream = ((cfg->reserved & 2u) || getenv("YDSCHED_FORCE_STREAM")) ? 1u : 0u;
  if (const char* e = getenv("YDSCHED_MERGE_CHUNK")) s->cfg_merge_chunk = std::max(32u, (uint32_t)atoi(e) & ~31u);
  if (const char* e = getenv("YDSCHED_MERGE_ROUNDS")) s->cfg_merge_rounds = std::max(2u, (uint32_t)atoi(e));
  s->tiny_ok = !(cfg->reserved & 4u) && !getenv("YDSCHED_NO_TINY");
  s->fused_cfg = !(cfg->reserved & 8u) && !getenv("YDSCHED_NO_FUSED");
  if (const char* e = getenv("YDSCHED_FUSED_MAX_N")) s->fused_max_nb = (uint32_t)std::max(1024, atoi(e));
  YD_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&s->h_fio), sizeof(yd::FusedHostIO), cudaHostAllocMapped));
  memset(s->h_fio, 0, sizeof(yd::FusedHostIO));
  YD_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&s->d_fio), s->h_fio, 0));
  s->host_prof = getenv("YDSCHED_HOST_PROF") != nullptr;
  s->fused_prof = getenv("YDSCHED_FUSED_PROF") != nullptr;
  {
    int sms = 0, per_sm = 0;
    YD_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device));
    YD_CUDA_CHECK(cudaFuncSetAttribute(yd::k_fused_front, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    YD_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, yd::k_fused_front, 1024, 64 * 1024));
    s->fused_grid = per_sm >= 1 ? (uint32_t)sms : 0u;  // (0: the kernel does not fit an SM -- never on sm_90a; the pipeline is used)
  }
  {
    const size_t prof_bytes = (yd::kProfHead + size_t(s->fused_grid) * yd::kProfBlockWords) * 8;
    s->d_fused_prof.ensure(prof_bytes);
    YD_CUDA_CHECK(cudaMemset(s->d_fused_prof.p, 0, prof_bytes));
  }
  s->debug_env = getenv("YDSCHED_DEBUG") != nullptr;
  YD_CUDA_CHECK(cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking));
  YD_CUDA_CHECK(cudaStreamCreateWithFlags(&s->st2, cudaStreamNonBlocking));
  YD_CUDA_CHECK(cudaStreamCreateWithFlags(&s->st_copy, cudaStreamNonBlocking));
  for (auto& e : s->ev) YD_CUDA_CHECK(cudaEventCreate(&e));
  for (auto& e : s->ev_f) YD_CUDA_CHECK(cudaEventCreate(&e));
  YD_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming));
  YD_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_join, cudaEventDisableTiming));
  YD_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_h2d, cudaEventDisableTiming));
  // (recorded again only after a request copy; the general graphs' wait nodes name it from their first capture on)
  YD_CUDA_CHECK(cudaEventRecord(s->ev_h2d, s->st_copy));
  YD_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_fin, cudaEventDisableTiming));
  s->ips.emplace_back();  // id 0 == YD_IP_NONE == the empty requestor string
  s->ip_ids.emplace("", 0);
  s->d_counters.ensure(sizeof(Counters));
  YD_CUDA_CHECK(cudaMemsetAsync(s->d_counters.p, 0, sizeof(Counters), s->st));
  s->h_counters.ensure(sizeof(Counters));
  s->h_small.ensure(1 << 16);
  s->d_dyn.ensure(sizeof(yd::DynParams));
  s->h_dyn.ensure(sizeof(yd::DynParams));
  s->h_fsc.ensure(sizeof(yd::FusedScalars));
  s->d_fsc.ensure(sizeof(yd::FusedScalars));
  s->h_meta.ensure(64);
  s->EnsureRing(0);
  return s;
}

void yd_destroy(yd_sched* s) {
  if (!s) return;
  yd_shard_finalize(s);
  cudaSetDevice(s->device);
  cudaStreamSynchronize(s->st);
  for (DevBuf* b : {&s->d_nproc, &s->d_load, &s->d_maxt, &s->d_flags, &s->d_ver, &s->d_run, &s->d_ever,
                    &s->d_run_tmp, &s->d_ever_tmp, &s->d_remap, &s->d_dec, &s->d_dec_tmp, &s->d_env_comp, &s->d_env_local,
                    &s->d_comp_sv_off, &s->d_comp_sv, &s->d_comp_mask_off, &s->d_comp_nwarps, &s->d_envmask,
                    &s->d_sv_comp, &s->d_sv_local, &s->d_ip_off, &s->d_ip_sv, &s->d_ip_comp_mask, &s->d_kept_env, &s->d_kept_sv,
                    &s->d_t_exp, &s->d_t_srv,
                    &s->d_t_flags, &s->d_reqs, &s->d_res, &s->d_out, &s->d_blk, &s->d_row_off, &s->d_row_len,
                    &s->d_codes, &s->d_ids, &s->d_ok, &s->d_counters, &s->d_sv_env_off, &s->d_sv_envs,
                    &s->d_comp_mode, &s->d_sv_emask, &s->d_slot_rec, &s->d_slot_spos, &s->d_slot_owner, &s->d_sort_k[0], &s->d_sort_k[1], &s->d_sort_v[0],
                    &s->d_sort_v[1], &s->d_zero, &s->d_list, &s->d_list_bal, &s->d_members, &s->d_rcls, &s->d_rrank, &s->d_rank_cnt, &s->d_rq, &s->d_rself,
                    &s->d_slot_pick, &s->d_mst_in, &s->d_mst_out, &s->d_stream_scratch, &s->d_reqs16, &s->d_out8, &s->d_fused_prof, &s->d_bloom,
                    &s->d_bloom_keys, &s->d_bloom_out, &s->d_rt_bytes, &s->d_rt_off, &s->d_rt_len, &s->d_rt_ids,
                    &s->d_rt_slots, &s->d_rt_keys, &s->d_rt_out}) {
    b->release();
  }
  for (auto& g : s->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (s->h_fio) cudaFreeHost(s->h_fio);
  s->d_dyn.release();
  s->d_fsc.release();
  for (PinBuf* b : {&s->h_facts, &s->h_topo, &s->h_counters, &s->h_small, &s->h_dyn, &s->h_meta, &s->h_fsc}) b->release();
  for (auto& e : s->ev) cudaEventDestroy(e);
  for (auto& e : s->ev_f) cudaEventDestroy(e);
  for (DevBuf* b : {&s->d_freqs, &s->d_fverdict, &s->d_ftile, &s->d_rpcs, &s->d_rpc_off, &s->d_rpc_ng, &s->d_rpc_res,
                    &s->d_rpc_out}) {
    b->release();
  }
  if (s->d_env_bytes) cudaFree(s->d_env_bytes);
  if (s->d_env_off) cudaFree(s->d_env_off);
  s->h_fcount.release();
  cudaEventDestroy(s->ev_fork); cudaEventDestroy(s->ev_join); cudaEventDestroy(s->ev_h2d); cudaEventDestroy(s->ev_fin);
  cudaStreamDestroy(s->st2); cudaStreamDestroy(s->st_copy);
  cudaStreamDestroy(s->st);
  delete s;
}

uint32_t yd_intern_env(yd_sched* s, const char* digest, size_t len) {
  return s->InternEnv(std::string(digest, len));
}
uint32_t yd_intern_ip(yd_sched* s, const char* ip, size_t len) { return s->InternIp(std::string(ip, len)); }

// KeepServantAlive, cc:190-220.  Pure registry work; the device copy of the facts
// is refreshed lazily before the next solve.
void yd_keep_servant_alive(yd_sched* s, int64_t now_ns, const yd_servant* v, int64_t expires_in_ns) {
  std::string loc = v->observed_location;
  auto it = s->loc2pos.find(loc);
  ServantHost* rec;
  std::vector<uint32_t> envs(v->num_envs);
  for (uint32_t i = 0; i != v->num_envs; ++i) envs[i] = s->InternEnv(v->env_digests[i]);
  if (it == s->loc2pos.end()) {
    s->loc2pos.emplace(loc, (uint32_t)s->sv.size());
    rec = &s->sv.emplace_back();
    rec->observed = loc;
    rec->discovered_at = now_ns;
    s->topo_dirty = true;
    s->order_dirty = true;
  } else {
    rec = &s->sv[it->second];
    if (rec->envs != envs) s->topo_dirty = true;
    uint32_t nf = 0;  // FactFlags of the new personality
    if (v->priority == YD_PRIORITY_DEDICATED) nf |= yd::kFlagDedicated;
    if (v->total_memory_in_bytes != 0 && v->memory_available_in_bytes < s->min_mem) nf |= yd::kFlagLowMem;
    if (rec->nproc != v->num_processors || rec->load != v->current_load || rec->max_tasks != v->max_tasks ||
        nf != s->FactFlags(*rec)) {
      s->order_dirty = true;  // a slot key or a free_end changed: the sorted slot order is rebuilt before the next solve
    }
  }
  rec->version = v->version;
  rec->reported = v->reported_location ? v->reported_location : "";
  rec->envs = std::move(envs);
  rec->nproc = v->num_processors;
  rec->load = v->current_load;
  rec->max_tasks = v->max_tasks;
  rec->total_mem = v->total_memory_in_bytes;
  rec->avail_mem = v->memory_available_in_bytes;
  rec->priority = v->priority;
  rec->reason = v->not_accepting_task_reason;
  rec->expires_at = now_ns + expires_in_ns;
  s->facts_dirty = true;
}

// ---- the two solvers' launch sequences -------------------------------------------

extern "C++" {
namespace {

constexpr size_t kRowscanMaxComponent = 32 * 32 * yd::kK;  // 8192 servants per component
constexpr size_t kStreamMaxComponent = 22000;              // 2 x u32 per servant of dynamic shared memory

yd::TopoView MakeTopo(yd_sched* s) {
  yd::TopoView t{};
  t.env_comp = s->d_env_comp.as<uint32_t>();
  t.n_envs = s->n_envs_dev;
  t.sv_comp = s->d_sv_comp.as<uint32_t>();
  t.sv_local = s->d_sv_local.as<uint32_t>();
  t.ip_off = s->d_ip_off.as<uint32_t>();
  t.ip_sv = s->d_ip_sv.as<uint32_t>();
  t.n_ips = s->n_ips_dev;
  t.sv_env_off = s->d_sv_env_off.as<uint32_t>();
  t.sv_envs = s->d_sv_envs.as<uint32_t>();
  t.comp_sv_off = s->d_comp_sv_off.as<uint32_t>();
  t.comp_sv = s->d_comp_sv.as<uint32_t>();
  t.sv_emask = s->emask_ok ? s->d_sv_emask.as<unsigned long long>() : nullptr;
  t.env_local = s->d_env_local.as<uint32_t>();
  t.ip_comp_mask = s->d_ip_comp_mask.as<unsigned long long>();
  return t;
}

yd::ClassTable MakeClassTable(yd_sched* s, const SolvePlan& plan) {
  uint32_t* u = reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_cls_off);
  yd::ClassTable ct{};
  // the 8-byte keys sit right behind res[] so one 0xFF memset initialises both
  ct.keys = reinterpret_cast<unsigned long long*>(s->d_res.as<uint32_t>() + s->res_words);
  ct.slot_cls = u;                       u += yd::kClsTableSize;
  ct.meta = u;                           u += 8;
  ct.cls_env = u;                        u += yd::kMaxClasses;
  ct.cls_mv = u;                         u += yd::kMaxClasses;
  ct.cls_comp = u;                       u += yd::kMaxClasses;
  ct.cls_nelig = u;                      u += yd::kMaxClasses;
  ct.cls_count = u;                      u += yd::kMaxClasses;
  ct.cls_lbit = u;                       u += yd::kMaxClasses;
  ct.comp_flags = u;                     u += s->n_comps;
  ct.comp_ncls = u;                      u += s->n_comps;
  ct.comp_midx = u;                      u += s->n_comps;
  ct.merge_comp = u;                     u += yd::kMaxClasses;
  ct.comp_cls = u;                       // [cls_bound * 32], the tail of the class region
  ct.cls_bound = s->cls_bound;
  ct.force_stream = plan.force_stream;
  return ct;
}

yd::MergePlan MakeMergePlan(yd_sched* s) {
  uint32_t* u = reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_merge_off);
  yd::MergePlan mp{};
  mp.bar = u;                            u += yd::kMaxClasses + 1;  // (only the first cell is used)
  mp.changed = u;                        u += 16;
  mp.dead = u;                           u += 16;
  mp.viol = u;                           u += s->n_comps;
  mp.tau = u;                            // [S]
  return mp;
}

// What the merge solver handed back in the last solve, for the YDSCHED_DEBUG lines: the OR of the components' yd::kBack*
// reasons, and how many components.  (Reads the scratch region: after the solve's sync, before the next solve.)
std::pair<uint32_t, uint32_t> MergeBack(yd_sched* s) {
  std::vector<uint32_t> viol(s->n_comps);
  YD_CUDA_CHECK(cudaMemcpy(viol.data(), MakeMergePlan(s).viol, viol.size() * 4, cudaMemcpyDeviceToHost));
  std::pair<uint32_t, uint32_t> r{0, 0};
  for (uint32_t v : viol) { r.first |= v; r.second += v != 0; }
  return r;
}

// Row-total mailboxes of the two row-parallel scans (k_scan_rows), in the zeroed scratch region.
unsigned long long* ScanPub(yd_sched* s, int which) {
  return reinterpret_cast<unsigned long long*>(static_cast<char*>(s->d_zero.p) + s->z_scan_off) + size_t(which) * (yd::kMaxClasses + 1);
}

yd::RqLayout MakeRqLayout(yd_sched* s, uint32_t q_base, uint32_t n_local, bool sharded) {
  uint32_t* u = reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_layout_off);
  yd::RqLayout L{};
  L.goff = u;                            u += yd::kMaxClasses;
  L.gn = u;                              u += yd::kMaxClasses;
  L.win = u;                             u += yd::kMaxClasses;
  L.base = u;                            u += yd::kMaxClasses;
  L.total = u;
  L.q_base = q_base;
  L.n_local = n_local;
  L.sharded = sharded ? 1u : 0u;
  L.rank_off = s->d_rank_cnt.as<uint32_t>();
  L.nrt = (uint32_t)((s->res_words + yd::kRankTile - 1) / yd::kRankTile);
  return L;
}

// Slot table (both solvers).  For the slot-stream solver it also records slot owners.
// Returns the number of kernels launched.
uint32_t LaunchSlotTable(yd_sched* s, bool for_stream, bool static_rows = false) {
  const uint32_t S = (uint32_t)s->sv.size();
  cudaStream_t st = s->st;
  yd::ServantArrays arr = s->arrays();
  const uint32_t sentinel = for_stream ? 0u : 1u;
  const uint32_t sr = static_rows ? 1u : 0u;
  yd::k_slot_rows<<<1, 1024, 0, st>>>(S, s->d_dyn.as<yd::DynParams>(), arr, s->d_row_off.as<uint32_t>(),
                                      s->d_row_len.as<uint32_t>(), s->d_counters.as<Counters>(), sentinel, sr);
  uint32_t* owner = for_stream ? s->d_slot_owner.as<uint32_t>() : nullptr;
  if (s->wide) {
    yd::k_slot_fill<true><<<(S + 7) / 8, 256, 0, st>>>(S, arr, s->d_row_off.as<uint32_t>(),
                                                       s->d_row_len.as<uint32_t>(), nullptr,
                                                       s->d_codes.as<unsigned long long>(), owner, sentinel, sr);
  } else {
    yd::k_slot_fill<false><<<(S + 7) / 8, 256, 0, st>>>(S, arr, s->d_row_off.as<uint32_t>(),
                                                        s->d_row_len.as<uint32_t>(), s->d_codes.as<uint32_t>(),
                                                        nullptr, owner, sentinel, sr);
  }
  return 2;
}

// Solver 1: one (task x servant) row per decision.
uint32_t LaunchRowscan(yd_sched* s) {
  cudaStream_t st = s->st;
  yd::SolveArgs a{};
  a.reqs = s->d_reqs.as<yd_task_req>();
  a.dp = s->d_dyn.as<yd::DynParams>();
  a.res = s->d_res.as<uint32_t>();
  a.env_comp = s->d_env_comp.as<uint32_t>();
  a.env_local = s->d_env_local.as<uint32_t>();
  a.n_envs = s->n_envs_dev;
  a.comp_sv_off = s->d_comp_sv_off.as<uint32_t>();
  a.comp_sv = s->d_comp_sv.as<uint32_t>();
  a.comp_mask_off = s->d_comp_mask_off.as<uint32_t>();
  a.comp_nwarps = s->d_comp_nwarps.as<uint32_t>();
  a.envmask = s->d_envmask.as<uint8_t>();
  a.sv_comp = s->d_sv_comp.as<uint32_t>();
  a.sv_local = s->d_sv_local.as<uint32_t>();
  a.ip_off = s->d_ip_off.as<uint32_t>();
  a.ip_sv = s->d_ip_sv.as<uint32_t>();
  a.n_ips = s->n_ips_dev;
  a.sv = s->arrays();
  a.row_off = s->d_row_off.as<uint32_t>();
  a.codes = s->d_codes.p;
  // Two register budgets: up to 8 solver warps (2048 servants per component) plus
  // 8 producer warps run with <= 128 registers per thread; larger components are
  // capped at 64 registers.
  const unsigned threads = std::min(32u, s->max_warps + yd::kMaxProducers) * 32;
  if (threads <= 512) {
    if (s->wide) yd::k_solve_rowscan<unsigned long long, 512><<<s->n_comps, threads, 0, st>>>(a);
    else yd::k_solve_rowscan<uint32_t, 512><<<s->n_comps, threads, 0, st>>>(a);
  } else {
    if (s->wide) yd::k_solve_rowscan<unsigned long long, 1024><<<s->n_comps, threads, 0, st>>>(a);
    else yd::k_solve_rowscan<uint32_t, 1024><<<s->n_comps, threads, 0, st>>>(a);
  }
  return 1;
}

template <typename KeyT>
uint32_t LaunchSort(yd_sched* s, int first_bit, int last_bit) {
  KeyT* const keys[2] = {s->d_sort_k[0].as<KeyT>(), s->d_sort_k[1].as<KeyT>()};
  uint32_t* const vals[2] = {s->d_sort_v[0].as<uint32_t>(), s->d_sort_v[1].as<uint32_t>()};
  return yd::rs_sort<KeyT>(s->d_codes.as<KeyT>(), &s->d_counters.as<Counters>()->slots, s->sort_nb, first_bit, last_bit,
                           reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_hist_off[0]), keys, vals,
                           s->st);
}

// Merge-solver chunk: more, shorter chunks pay while the request-side passes are short (measured on an H100 SXM, 700 W:
// cfg2-random 324 vs 374 us, cfg-self 177 vs 187 us at 256 vs 512 slots; cfg3, 1 M requests, 604 vs 573 us).  A sharded
// solve keeps one length whatever each rank's batch.
uint32_t MergeChunk(const yd_sched* s, uint32_t Nb) {
  if (s->cfg_merge_chunk) return s->cfg_merge_chunk;
  return !s->shard && Nb <= 262144 ? 256u : 512u;
}

// (class, slot) entries the slot lists hold per slot: a batch whose classes are eligible on more slots than that
// overflows them (flag 1) and is decided by the row-scan solver.
constexpr size_t kListEntriesPerSlot = 4;

// The per-solve buffers of size class (Nb, slot_b) that both solvers and the sharded solve use.
void EnsureSolveBuffers(yd_sched* s, uint32_t Nb, size_t slot_b) {
  s->d_reqs.ensure(size_t(Nb) * sizeof(yd_task_req));
  s->res_words = Nb;
  s->d_res.ensure(size_t(Nb) * 4 + yd::kClsTableSize * 8);
  s->d_out.ensure(size_t(Nb) * sizeof(yd_grant));
  s->d_blk.ensure(size_t((Nb + 1023) / 1024) * 4);
  s->d_row_off.ensure((s->sv.size() + 1) * 4);
  s->d_row_len.ensure((s->sv.size() + 1) * 4);
  s->d_codes.ensure(slot_b * (s->wide ? 8 : 4));
  s->d_slot_owner.ensure(slot_b * 4);
}

// The call's scalars, in the host copy the solve uploads.
const yd::DynParams& SetDynParams(yd_sched* s, uint32_t n, uint32_t slot_clamp, int64_t now_ns) {
  return *s->h_dyn.as<yd::DynParams>() = yd::DynParams{n, slot_clamp, now_ns, s->lo, s->next_id};
}

// Flag 2 (more lists than provisioned): one list per class plus one pseudo-class list per merge-mode component are
// needed, so the class bound doubles until it holds them, up to kMaxClasses.  False when it is there already.
bool GrowClassBound(yd_sched* s, const uint32_t* meta) {
  if (s->cls_bound >= yd::kMaxClasses) return false;
  const uint32_t want = meta[0] + meta[2] + 1;
  s->cls_bound *= 2;
  while (s->cls_bound < want && s->cls_bound < yd::kMaxClasses) s->cls_bound *= 2;
  return true;
}

// Allocates everything the slot-stream sequence touches for size class (Nb, slot_b) and
// lays out the zero-initialised scratch region; called before a graph capture so that no
// allocation happens inside it.
void PrepareStreamBuffers(yd_sched* s, uint32_t Nb, size_t slot_b) {
  const size_t ksz = s->wide ? 8 : 4;
  for (int b = 0; b < 2; ++b) { s->d_sort_k[b].ensure(slot_b * ksz); s->d_sort_v[b].ensure(slot_b * 4); }
  s->d_slot_rec.ensure(slot_b * 8);
  s->d_slot_spos.ensure(slot_b * 4);
  s->sort_nb = (uint32_t)((slot_b + yd::kRsTile - 1) / yd::kRsTile);
  const int passes = s->wide ? 9 : 4;
  size_t off = 0;
  for (int p = 0; p < passes; ++p) { s->z_hist_off[p] = off; off += yd::rs_pass_words(s->sort_nb) * 4; }
  s->z_cls_off = off;
  off += (yd::kClsTableSize + 8 + 7 * yd::kMaxClasses + 3 * size_t(s->n_comps) + 32 * size_t(s->cls_bound) + 8) * 4;
  s->z_merge_off = off;
  off += (yd::kMaxClasses + 1 + 32 + size_t(s->n_comps) + s->sv.size() + 8) * 4;
  s->z_layout_off = off;
  off += (4 * yd::kMaxClasses + 8) * 4;
  off = (off + 7) & ~size_t(7);
  s->z_scan_off = off;
  off += 2 * (yd::kMaxClasses + 1) * 8;
  s->z_final_off = off;
  off += (size_t(Nb + 1023) / 1024 + 2) * 8;
  s->z_fbar_off = off;
  off += 8 * 4;
  const uint32_t n_tiles = (uint32_t)((slot_b + yd::kListTile - 1) / yd::kListTile);
  s->z_listcnt_off = off;
  off += (size_t(s->cls_bound) * n_tiles + 1) * 4;
  s->z_bytes = (off + 255) & ~size_t(255);
  s->d_zero.ensure(s->z_bytes);
  s->d_list.ensure(slot_b * kListEntriesPerSlot * sizeof(uint2));
  s->d_list_bal.ensure(size_t(n_tiles) * s->cls_bound * 32 * 4);  // membership ballots: (tile, list, warp)
  // member lists of the fused solo solve: (tile, list, rank in the tile), for the batches the fused kernel may take --
  // cls_bound x tiles <= 32768, so 128 MiB at most (allocated here, before the scratch signature is taken: a buffer
  // that grew on a steady call would bump g_buf_generation and cost the next solve its speculation)
  if (s->fused_cfg && Nb <= s->fused_max_nb && size_t(s->cls_bound) * n_tiles <= 32768) {
    s->d_members.ensure(size_t(n_tiles) * s->cls_bound * yd::kListTile * 4);
  }
  const uint32_t n_rtiles = (Nb + yd::kRankTile - 1) / yd::kRankTile;
  s->d_rcls.ensure(size_t(Nb) * 4); s->d_rrank.ensure(size_t(Nb) * 4); s->d_rq.ensure(size_t(Nb) * 8);
  s->d_rself.ensure(size_t(Nb) * 4);
  s->d_stream_scratch.ensure(std::max<size_t>(s->sv.size(), 1) * 8);
  s->d_slot_pick.ensure(slot_b * kListEntriesPerSlot * 4);  // one word per list entry
  // every slot is in at most one pseudo-class list: chunks <= slots / chunk + one partial chunk per list
  s->merge_max_chunks = (uint32_t)(slot_b / MergeChunk(s, Nb)) + s->cls_bound + 1;
  s->d_mst_in.ensure(size_t(s->merge_max_chunks) * yd::kMergeStateWords * 4);
  s->d_mst_out.ensure(size_t(s->merge_max_chunks) * yd::kMergeStateWords * 4);
  s->d_rank_cnt.ensure((size_t(s->cls_bound) * n_rtiles + 1) * 4);
  if (!s->stream_attr_set) {
    YD_CUDA_CHECK(cudaFuncSetAttribute(yd::k_solve_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, 190 * 1024));
    s->stream_attr_set = true;
  }
}

// The tiling of one solve attempt of size class (Nb, slot_b), and its list counts in the zeroed scratch region (laid out
// by PrepareStreamBuffers, so built after it).
struct SolveGeometry {
  uint32_t n_ltiles, n_rtiles;  // slot tiles (kListTile slots), request tiles (kRankTile requests)
  size_t list_cap;              // entries of d_list
  uint32_t* list_cnt;           // (class, slot tile) list counts
};

SolveGeometry MakeGeometry(yd_sched* s, uint32_t Nb, size_t slot_b) {
  return SolveGeometry{(uint32_t)((slot_b + yd::kListTile - 1) / yd::kListTile), (Nb + yd::kRankTile - 1) / yd::kRankTile,
                       slot_b * kListEntriesPerSlot,
                       reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_listcnt_off)};
}

// On `st`, after k_cls_insert: the final class table, each class's eligible servants, and the requests' FIFO ranks with
// their scan.  `ev_fin` (if any) is recorded as soon as the class table is final.  Returns the kernels launched.
uint32_t LaunchClassPhase(yd_sched* s, const SolveGeometry& g, const yd::TopoView& t, const yd::ClassTable& ct,
                          cudaStream_t st, cudaEvent_t ev_fin) {
  const yd::ServantArrays arr = s->arrays();
  yd::k_cls_finalize<<<1, 1024, 0, st>>>(t, ct, arr, s->n_comps, s->d_comp_mode.as<uint32_t>());
  if (ev_fin) YD_CUDA_CHECK(cudaEventRecord(ev_fin, st));
  yd::k_cls_elig<<<ct.cls_bound, 256, 0, st>>>(t, ct, arr);
  yd::k_rank_count<<<g.n_rtiles, yd::kRankTile, 0, st>>>(s->d_reqs.as<yd_task_req>(), s->d_dyn.as<yd::DynParams>(), t, ct,
                                                          s->d_comp_mode.as<uint32_t>(), g.n_rtiles,
                                                          s->d_rcls.as<uint32_t>(), s->d_rrank.as<uint32_t>(),
                                                          s->d_rself.as<uint32_t>(), s->d_rank_cnt.as<uint32_t>());
  yd::k_scan_rows<<<ct.cls_bound, 1024, 0, st>>>(s->d_rank_cnt.as<uint32_t>(), ct.meta, g.n_rtiles, ScanPub(s, 0));
  return 4;
}

// On `st`, once the class table is final: the per-class slot lists, read through `dec`.  Returns the kernels launched.
uint32_t LaunchListPhase(yd_sched* s, const SolveGeometry& g, const yd::SlotDecode& dec, const yd::TopoView& t,
                         const yd::ClassTable& ct, cudaStream_t st) {
  const unsigned long long* m_ptr = &s->d_counters.as<Counters>()->slots;
  yd::k_list_count<<<g.n_ltiles, yd::kListTile, 0, st>>>(m_ptr, dec, t, ct, s->arrays(), g.n_ltiles, g.list_cnt,
                                                         s->d_list_bal.as<uint32_t>());
  yd::k_scan_rows<<<ct.cls_bound, 1024, 0, st>>>(g.list_cnt, ct.meta + 3, g.n_ltiles, ScanPub(s, 1));
  yd::k_list_fill<<<g.n_ltiles, yd::kListTile, 0, st>>>(m_ptr, dec, t, ct, g.n_ltiles, g.list_cnt,
                                                        s->d_list_bal.as<uint32_t>(), s->d_list.as<uint2>(),
                                                        (uint32_t)g.list_cap);
  return 3;
}

// The merge solver's arguments; LaunchMerge adds its launch shape.
yd::MergeArgs MakeMergeArgs(yd_sched* s, const SolveGeometry& g, const yd::ClassTable& ct, const yd::RqLayout& L) {
  yd::MergeArgs m{};
  m.t = MakeTopo(s); m.ct = ct; m.mp = MakeMergePlan(s); m.sv = s->arrays(); m.dp = s->d_dyn.as<yd::DynParams>();
  m.comp_mode = s->d_comp_mode.as<uint32_t>();
  m.list_off = g.list_cnt; m.n_list_tiles = g.n_ltiles; m.list = s->d_list.as<uint2>();
  m.rank_off = s->d_rank_cnt.as<uint32_t>(); m.n_rank_tiles = g.n_rtiles;
  m.rq = s->d_rq.as<uint2>(); m.rcls = s->d_rcls.as<uint32_t>(); m.rself = s->d_rself.as<uint32_t>();
  m.slot_pick = s->d_slot_pick.as<uint32_t>();
  m.st_in = s->d_mst_in.as<uint32_t>(); m.st_out = s->d_mst_out.as<uint32_t>();
  m.res = s->d_res.as<uint32_t>();
  m.L = L;
  return m;
}

// The merge solver: ONE persistent launch (rounds, scatter and check are phases behind grid barriers), so the
// grid must be co-resident: occupancy x SMs blocks at most, each looping over its chunks.
uint32_t LaunchMerge(yd_sched* s, uint32_t Nb, yd::MergeArgs& m, cudaStream_t st) {
  m.kcap = std::min(32u, s->cls_bound);
  const size_t dyn = size_t(1 + m.kcap) * yd::kRingRecs * sizeof(uint2);
  if (s->merge_grid_kcap != m.kcap) {
    int per_sm = 0, sms = 0;
    YD_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, yd::k_merge_solve, 32, dyn));
    YD_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device));
    s->merge_grid = (uint32_t)std::max(1, std::min(per_sm, 16) * sms);
    s->merge_grid_kcap = m.kcap;
  }
  m.chunk = MergeChunk(s, Nb);
  m.max_chunks = s->merge_max_chunks;
  m.diag = &s->d_counters.as<Counters>()->pad[0];
  m.rq_blocks = (uint32_t)(s->d_rq.cap / 256);
  m.ls_blocks = (uint32_t)(s->d_list.cap / 256);
  const uint32_t grid = std::min(s->merge_grid, s->merge_max_chunks);
  yd::k_merge_solve<<<grid, 32, dyn, st>>>(m);
  yd::k_merge_check<<<(std::max(m.L.n_local, 1u) + 255) / 256, 256, 0, st>>>(m);
  return 2;
}

constexpr size_t kStaticSlotLimit = size_t(1) << 26;

// (Re)builds the kept slot order: slot table over ALL running_tasks values + its sort, outside any graph.
// Buffers must exist (PrepareStreamBuffers).  Returns the number of kernels launched.
uint32_t RebuildSlotOrder(yd_sched* s, size_t slot_b) {
  cudaStream_t st = s->st;
  // the sort's digit histograms live in the zeroed scratch region
  YD_CUDA_CHECK(cudaMemsetAsync(static_cast<char*>(s->d_zero.p) + s->z_hist_off[0], 0, s->z_cls_off - s->z_hist_off[0], st));
  uint32_t l = LaunchSlotTable(s, true, true);
  if (s->wide) l += LaunchSort<unsigned long long>(s, 0, 62);
  else l += LaunchSort<uint32_t>(s, 3, 30);
  {
    yd::SlotDecode dec{s->d_sort_v[0].as<uint32_t>(), s->d_slot_owner.as<uint32_t>(), s->d_row_off.as<uint32_t>(),
                       s->d_row_len.as<uint32_t>(), s->d_run.as<uint32_t>(), 1u, nullptr};
    yd::k_slot_records<<<(unsigned)((slot_b + 255) / 256), 256, 0, st>>>(&s->d_counters.as<Counters>()->slots, dec,
                                                                          s->d_slot_rec.as<uint2>(),
                                                                          s->d_slot_spos.as<uint32_t>());
    l += 1;
  }
  YD_CUDA_CHECK(cudaGetLastError());
  s->order_dirty = false;
  s->order_static = true;
  s->order_slot_b = slot_b;
  s->order_rebuilds += 1;
  return l;
}

// The solvers for everything the data-parallel path does not decide: the merge solver (all components but those with
// several servants behind one requestor IP), then the sequential slot-stream walk for the rest.
uint32_t LaunchCoupledSolvers(yd_sched* s, uint32_t N, const SolveGeometry& g, const SolvePlan& plan, const yd::RqLayout& L) {
  cudaStream_t st = s->st;
  // ---- merge solver: everything but components with several servants behind one requestor IP -------
  yd::MergeArgs m = MakeMergeArgs(s, g, MakeClassTable(s, plan), L);
  const uint32_t launches = LaunchMerge(s, N, m, st);

  // ---- sequential decisions for everything else ---------------------------------------------
  yd::StreamArgs a{};
  a.reqs = s->d_reqs.as<yd_task_req>();
  a.dp = m.dp;
  a.res = s->d_res.as<uint32_t>();
  a.t = m.t;
  a.ct = m.ct;
  a.sv = m.sv;
  a.row_len = s->d_row_len.as<uint32_t>();
  a.static_rows = s->order_static ? 1u : 0u;
  a.list_off = g.list_cnt;
  a.n_list_tiles = g.n_ltiles;
  a.list = s->d_list.as<uint2>();
  a.max_comp_servants = (uint32_t)std::min<size_t>(s->max_comp_servants, kStreamMaxComponent);
  a.gscratch = s->d_stream_scratch.as<uint32_t>();
  a.n_servants = (uint32_t)s->sv.size();
  a.comp_mode = s->d_comp_mode.as<uint32_t>();
  a.viol = m.mp.viol;
  a.counters = s->d_counters.as<Counters>();
  const size_t dyn = size_t(a.max_comp_servants) * 8;
  yd::k_solve_stream<<<s->n_comps, (yd::kStreamProducers + 1) * 32, dyn, st>>>(a);
  return launches + 1;
}

// `st` waits for the request upload on the copy stream: when this call copied requests (`copied`), and always in a
// capture, whose graph is replayed by calls that copy and calls that do not.  A staged or zero-copy solve outside a graph
// has nothing to wait for.  `capturing` selects the external-event flavour (the upload is never part of a graph).
void WaitUpload(yd_sched* s, cudaStream_t st, bool copied, bool capturing) {
  if (copied || capturing) YD_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_h2d, capturing ? cudaEventWaitExternal : 0));
}

// Solver 2: sorted slot streams.  Two concurrent branches:
//   st  : slot table (+ first histogram) -> radix passes
//   st2 : [wait for the request upload] class table -> finalize -> FIFO ranks -> scan
// joined before the per-class lists.
uint32_t LaunchStream(yd_sched* s, uint32_t N, const SolveGeometry& g, const SolvePlan& plan, bool copied, bool capturing) {
  cudaStream_t st = s->st, st2 = s->st2;
  uint32_t launches = 0;
  yd::TopoView t = MakeTopo(s);
  yd::ClassTable ct = MakeClassTable(s, plan);
  yd::ServantArrays arr = s->arrays();
  const yd::DynParams* dp = s->d_dyn.as<yd::DynParams>();

  // ---- fork ---------------------------------------------------------------------
  YD_CUDA_CHECK(cudaEventRecord(s->ev_fork, st));
  YD_CUDA_CHECK(cudaStreamWaitEvent(st2, s->ev_fork, 0));
  // branch B: classes and FIFO ranks (needs the requests in HBM)
  WaitUpload(s, st2, copied, capturing);
  yd::k_cls_insert<<<(N + 255) / 256, 256, 0, st2>>>(s->d_reqs.as<yd_task_req>(), dp, t, ct);
  launches += 1 + LaunchClassPhase(s, g, t, ct, st2, s->ev_fin);  // (the list kernels on `st` wait for ev_fin alone)
  YD_CUDA_CHECK(cudaEventRecord(s->ev_join, st2));
  // branch A: slot table and its sort -- unless the kept (static) order is valid
  if (!s->order_static) {
    launches += LaunchSlotTable(s, true);
    if (s->wide) launches += LaunchSort<unsigned long long>(s, 0, 62);
    else launches += LaunchSort<uint32_t>(s, 3, 30);
  }
  YD_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_fin, 0));

  // ---- per-class sorted slot lists ----------------------------------------------------
  const yd::SlotDecode dec{s->d_sort_v[0].as<uint32_t>(), s->d_slot_owner.as<uint32_t>(), s->d_row_off.as<uint32_t>(),
                           s->d_row_len.as<uint32_t>(), s->d_run.as<uint32_t>(), s->order_static ? 1u : 0u,
                           s->order_static ? s->d_slot_rec.as<uint2>() : nullptr};
  launches += LaunchListPhase(s, g, dec, t, ct, st);

  // ---- join: FIFO ranks and eligibility counts are needed from here on ---------------------------------------
  YD_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_join, 0));
  // ---- data-parallel path: single-class components without self-requests ----------------
  // (n_local = the grid bound: res[] has that many cells and only requests < dp->n are ever named)
  const yd::RqLayout L = MakeRqLayout(s, 0, N, false);
  yd::k_rank_assign<<<(N + 255) / 256, 256, 0, st>>>(dp, g.n_rtiles, t, ct, s->d_rcls.as<uint32_t>(),
                                                     s->d_rrank.as<uint32_t>(), s->d_rself.as<uint32_t>(),
                                                     s->d_rank_cnt.as<uint32_t>(), g.list_cnt,
                                                     g.n_ltiles, s->d_list.as<uint2>(), arr, s->d_comp_mode.as<uint32_t>(),
                                                     s->d_rq.as<uint2>(), s->d_res.as<uint32_t>(), L);
  launches += 1;

  launches += LaunchCoupledSolvers(s, N, g, plan, L);
  return launches;
}

// The solo kernel searches the scanned list offsets, cls_bound x (slot tiles + 1) + 1 words, once per request.  When they
// fit in dynamic shared memory (64 KB at most) every block derives the offsets it needs from the raw counts, without
// the leader scans of E2 (fused.cuh); the speculative variant needs that.  Returns the words, 0 when they do not fit.
uint32_t FusedLoffWords(const yd_sched* s, const SolveGeometry& g) {
  const size_t cells = size_t(s->cls_bound) * (g.n_ltiles + 1) + 1;
  return cells <= 16384 ? (uint32_t)cells : 0u;
}

// The arguments of the fused front kernel (fused.cuh) for a batch of size class N.  `capturing` (general variants only):
// the scalars come through a copy node enqueued here; a solo launch, never graphed, gets them as kernel parameters.
yd::FusedArgs MakeFusedArgs(yd_sched* s, uint32_t N, const SolveGeometry& g, const SolvePlan& plan, bool capturing,
                            bool packed_in, bool packed_out) {
  const bool solo = IsSolo(plan.variant);
  yd::FusedArgs a{};
  a.sc = s->fsc;
  a.sc_dev = (capturing && !solo) ? s->d_fsc.as<yd::FusedScalars>() : nullptr;
  if (a.sc_dev) YD_CUDA_CHECK(cudaMemcpyAsync(s->d_fsc.p, s->h_fsc.p, sizeof(yd::FusedScalars), cudaMemcpyHostToDevice, s->st));
  a.hio = s->d_fio;
  a.dyn_out = solo ? nullptr : s->d_dyn.as<yd::DynParams>();
  a.clean_keys = reinterpret_cast<unsigned long long*>(s->d_res.as<uint32_t>() + s->res_words);
  a.clean_zero = reinterpret_cast<uint4*>(static_cast<char*>(s->d_zero.p) + s->z_cls_off);
  a.clean_zero_vec = (uint32_t)((s->z_bytes - s->z_cls_off) / 16);
  a.reqs = s->d_reqs.as<yd_task_req>();
  a.reqs16 = packed_in ? s->d_reqs16.as<uint4>() : nullptr;
  a.reqs16_w = packed_in ? s->d_reqs16.as<uint4>() : nullptr;
  a.reqs_w = (packed_in && !solo) ? s->d_reqs.as<yd_task_req>() : nullptr;
  a.t = MakeTopo(s);
  a.ct = MakeClassTable(s, plan);
  a.sv = s->arrays();
  a.dec = yd::SlotDecode{s->d_sort_v[0].as<uint32_t>(), s->d_slot_owner.as<uint32_t>(), s->d_row_off.as<uint32_t>(),
                         s->d_row_len.as<uint32_t>(), s->d_run.as<uint32_t>(), 1u, s->d_slot_rec.as<uint2>()};
  a.m_ptr = &s->d_counters.as<Counters>()->slots;
  a.comp_mode = s->d_comp_mode.as<uint32_t>();
  a.n_comps = s->n_comps;
  a.n_rtiles = g.n_rtiles;
  a.n_ltiles = g.n_ltiles;
  a.rcls = s->d_rcls.as<uint32_t>();
  a.rrank = s->d_rrank.as<uint32_t>();
  a.rself = s->d_rself.as<uint32_t>();
  a.rank_cnt = s->d_rank_cnt.as<uint32_t>();
  a.list_cnt = g.list_cnt;
  a.list_bal = s->d_list_bal.as<uint32_t>();
  a.members = s->d_members.as<uint32_t>();
  a.list = s->d_list.as<uint2>();
  a.list_cap = (uint32_t)g.list_cap;
  a.rq = s->d_rq.as<uint2>();
  a.res = s->d_res.as<uint32_t>();
  a.L = MakeRqLayout(s, 0, N, false);
  a.bar = reinterpret_cast<uint32_t*>(static_cast<char*>(s->d_zero.p) + s->z_fbar_off);
  a.solo = solo ? 1u : 0u;
  a.packed_out = packed_out ? 1u : 0u;
  a.comp_sv = s->d_comp_sv.as<uint32_t>();
  a.ring = s->ring();
  a.out = packed_out ? s->d_out8.p : s->d_out.p;
  a.counters = s->d_counters.as<Counters>();
  a.n_servants = (uint32_t)s->sv.size();
  a.prof = s->fused_prof ? s->d_fused_prof.as<unsigned long long>() : nullptr;
  a.loff_cache_words = solo ? FusedLoffWords(s, g) : 0u;
  a.spec = plan.variant == kSoloSpec ? 1u : 0u;
  a.kept_env = s->d_kept_env.as<uint4>();
  a.kept_sv = s->d_kept_sv.as<uint32_t>();
  a.slot_spos = s->d_slot_spos.as<uint32_t>();
  return a;
}

// The fused front kernel on `st`, one block per SM whatever the batch (the phases hand out tiles of two kinds): classes,
// ranks, lists and the data-parallel verdicts in ONE persistent launch; solo variants: grants, task ids and leases too
// (batches made of data-parallel components only).  Needs the kept slot order.
void LaunchFusedKernel(yd_sched* s, const yd::FusedArgs& a) {
  yd::k_fused_front<<<s->fused_grid, 1024, size_t(a.loff_cache_words) * 4, s->st>>>(a);
}

// A general (not solo) fused solve: the fused front kernel, then the coupled solvers.
uint32_t LaunchFused(yd_sched* s, uint32_t N, const SolveGeometry& g, const SolvePlan& plan, bool copied, bool capturing,
                     bool packed_in, bool packed_out) {
  const yd::FusedArgs a = MakeFusedArgs(s, N, g, plan, capturing, packed_in, packed_out);
  WaitUpload(s, s->st, copied, capturing);
  LaunchFusedKernel(s, a);
  return 1 + LaunchCoupledSolvers(s, N, g, plan, a.L);
}

}  // namespace
}  // extern "C++"

extern "C++" {
namespace {

uint64_t NextPow2(uint64_t v, uint64_t lo) {
  uint64_t r = lo;
  while (r < v) r <<= 1;
  return r;
}

// What turns the packed grants of the next batch into task ids (yd_packed_ids): its first task id and the stride.
yd_packed_ids BatchIds(const yd_sched* s) { return yd_packed_ids{s->next_id * s->id_stride + s->id_offset, s->id_stride}; }

// One call decides at most 2^30 requests (packed grant ordinals have 30 bits).
void CheckBatchSize(size_t n) {
  if (n > 0x40000000ull) { fprintf(stderr, "ydsched: batch too large\n"); abort(); }
}

// yd_last_solve_stats reports zeros from here on, until the caller fills fields in.
void ResetStats(yd_sched* s) { s->stats = yd_solve_stats{}; s->stats_times_pending = 0; s->have_stats = true; }

// n requests as 24-byte records: copied from `reqs`, or unpacked from `reqs16`.
void CopyRequests(const yd_task_req* reqs, const yd_task_req16* reqs16, size_t n, yd_task_req* r) {
  if (reqs) memcpy(r, reqs, n * sizeof(yd_task_req));
  else for (size_t i = 0; i != n; ++i) r[i] = yd_unpack_req(reqs16[i]);
}

// n grants to the caller: 16-byte records to `out`, or packed with the batch's `ids` to `out8`.
void WriteGrants(yd_grant* out, yd_grant8* out8, const yd_packed_ids& ids, const yd_grant* g, size_t n) {
  if (out8) for (size_t i = 0; i != n; ++i) out8[i] = yd_pack_grant(g[i], ids);
  else if (n) memcpy(out, g, n * sizeof(yd_grant));
}

// n grants packed with `ids` into d_out8, for a device-side consumer (`keep8` of WaitImpl and ShardSolve): the grants
// of the paths that decide on the host side of the device (halves, the group's whole-queue fallback, no servants).
void UploadGrants8(yd_sched* s, const yd_packed_ids& ids, const yd_grant* g, size_t n) {
  if (!n) return;
  std::vector<yd_grant8> g8(n);
  for (size_t i = 0; i != n; ++i) g8[i] = yd_pack_grant(g[i], ids);
  s->d_out8.ensure(n * sizeof(yd_grant8));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_out8.p, g8.data(), n * sizeof(yd_grant8), cudaMemcpyHostToDevice, s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
}

// Everything between the request upload and the grant download, for size class (Nb, slot_b), of a general (not solo)
// solve: the sequence that is captured into a CUDA graph.  (A solo solve is one kernel: LaunchSolo launches it.)
// packed bit 0: the upload is 16-byte records in d_reqs16; bit 1: the download is 8-byte grants from d_out8.
// `copied`: this call copied the requests on the copy stream (WaitUpload).
uint32_t EnqueueSolve(yd_sched* s, uint32_t Nb, const SolveGeometry& g, const SolvePlan& plan, bool record_events,
                      bool copied, bool capturing, uint32_t packed) {
  cudaStream_t st = s->st;
  const uint32_t S = (uint32_t)s->sv.size();
  const uint32_t solver = plan.solver;
  const bool have_work = S && s->n_comps;
  const uint32_t nb = (Nb + 1023) / 1024;
  const bool packed_in = packed & 1u, packed_out = packed & 2u;
  uint32_t launches = 0;
  const yd::DynParams* dp = s->d_dyn.as<yd::DynParams>();
  const bool fused = plan.variant != kPipeline && have_work && solver == 2;
  // (the fused kernel reads the call's scalars from its parameters or d_fsc and stores them in d_dyn itself)
  if (!fused) YD_CUDA_CHECK(cudaMemcpyAsync(s->d_dyn.p, s->h_dyn.p, sizeof(yd::DynParams), cudaMemcpyHostToDevice, st));
  // res[] = kResEnvNotFound, and (slot-stream) the class-table keys behind it = empty
  YD_CUDA_CHECK(cudaMemsetAsync(s->d_res.p, 0xFF, size_t(Nb) * 4 + (solver == 2 ? yd::kClsTableSize * 8 : 0), st));
  if (solver == 2 && have_work) YD_CUDA_CHECK(cudaMemsetAsync(s->d_zero.p, 0, s->z_bytes, st));
  if (record_events) YD_CUDA_CHECK(cudaEventRecord(s->ev[1], st));
  const uint32_t* abort_flag = nullptr;
  if (packed_in && !fused) {
    // 16-byte upload -> the 24-byte queue the pipeline kernels read
    WaitUpload(s, st, copied, capturing);
    yd::k_unpack_reqs<<<(Nb + 255) / 256, 256, 0, st>>>(s->d_reqs16.as<uint4>(), dp, s->d_reqs.as<yd_task_req>());
    launches += 1;
  }
  if (have_work && solver == 2) {
    if (record_events) YD_CUDA_CHECK(cudaEventRecord(s->ev[2], st));
    if (fused) launches += LaunchFused(s, Nb, g, plan, copied, capturing, packed_in, packed_out);
    else launches += LaunchStream(s, Nb, g, plan, copied, capturing);
    abort_flag = MakeClassTable(s, plan).meta + 1;
  } else {
    if (have_work) launches += LaunchSlotTable(s, false);
    if (record_events) YD_CUDA_CHECK(cudaEventRecord(s->ev[2], st));
    // the row-scan kernels read the requests: they were uploaded on the copy stream
    WaitUpload(s, st, copied, capturing);
    if (have_work) launches += LaunchRowscan(s);
  }
  if (record_events) YD_CUDA_CHECK(cudaEventRecord(s->ev[3], st));
  if (solver == 2 && have_work && nb <= 2048) {
    // grants, task ids (single-pass scan with look-back), leases, ++running_tasks: one launch (beyond ~2 M requests the
    // look-back chain of 1024-thread blocks is slower than three plain passes)
    unsigned long long* look = reinterpret_cast<unsigned long long*>(static_cast<char*>(s->d_zero.p) + s->z_final_off);
    yd::k_final_fused<<<nb, 1024, 0, st>>>(s->d_res.as<uint32_t>(), s->d_reqs.as<yd_task_req>(), dp, look, nb,
                                           s->d_comp_sv.as<uint32_t>(), s->ring(), s->d_out.as<yd_grant>(),
                                           s->d_counters.as<Counters>(), abort_flag, s->d_run.as<uint32_t>(),
                                           s->d_ever.as<unsigned long long>());
    launches += 1;
  } else {
    yd::k_final_count<<<nb, 1024, 0, st>>>(s->d_res.as<uint32_t>(), dp, s->d_blk.as<uint32_t>(), abort_flag);
    yd::k_final_scan<<<1, 1024, 0, st>>>(s->d_blk.as<uint32_t>(), nb, s->d_counters.as<Counters>(), abort_flag);
    yd::k_final_write<<<nb, 1024, 0, st>>>(s->d_res.as<uint32_t>(), s->d_reqs.as<yd_task_req>(), dp,
                                           s->d_blk.as<uint32_t>(), s->d_comp_sv.as<uint32_t>(), s->ring(),
                                           s->d_out.as<yd_grant>(), abort_flag,
                                           // the row-scan solver writes running_tasks back itself
                                           solver == 2 ? s->d_run.as<uint32_t>() : nullptr,
                                           s->d_ever.as<unsigned long long>());
    launches += 3;
  }
  if (packed_out) {
    yd::k_pack_grants<<<(Nb + 255) / 256, 256, 0, st>>>(s->d_out.as<uint4>(), dp, s->ring(), s->d_out8.as<uint2>());
    launches += 1;
  }
  YD_CUDA_CHECK(cudaGetLastError());
  if (record_events) YD_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->h_counters.p, s->d_counters.p, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  if (abort_flag) {
    YD_CUDA_CHECK(cudaMemcpyAsync(s->h_meta.p, abort_flag - 1, 32, cudaMemcpyDeviceToHost, st));  // meta[0..7]
  }
  return launches;
}

}  // namespace
}  // extern "C++"

// THE HOT PATH: n sequential WaitForStartingNewTask decisions (cc:93-140).
// Queue staging: a front end can move the pending queue into HBM while RPCs are still
// arriving and start the solve when the batch closes.
void yd_stage_requests(yd_sched* s, const yd_task_req* reqs, size_t n) {
  CheckBatchSize(n);
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->staged_n = 0;
  if (n == 0) return;
  s->d_reqs.ensure(size_t(NextPow2(n, 1024)) * sizeof(yd_task_req));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_reqs.p, reqs, n * sizeof(yd_task_req), cudaMemcpyHostToDevice, s->st_copy));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st_copy));  // `reqs` may be reused by the caller right away
  s->staged_n = n;
}

void yd_wait_for_staged_tasks(yd_sched* s, int64_t now_ns, size_t n, yd_grant* out) {
  if (n == 0) return;
  if (n > s->staged_n) { fprintf(stderr, "ydsched: %zu requests asked for, %zu staged\n", n, s->staged_n); abort(); }
  yd_wait_for_starting_new_tasks(s, now_ns, nullptr, n, out);
}

extern "C++" {
namespace {
// YDSCHED_HOST_PROF: host-side timestamps of a solve (microseconds; 0 when off), printed at its end.
struct HostProf {
  bool on;
  double t[8] = {};
  void Stamp(int i) { if (on) t[i] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
  void Print() {
    if (!on) return;
    Stamp(7);
    fprintf(stderr, "ydsched: host us: prep %.1f (attrs+variant %.1f) upload+prep %.1f launch %.1f d2h-enqueue %.1f sync-wait %.1f stats %.1f total %.1f\n",
            t[1] - t[0], t[2] - t[1], t[3] - t[2], t[4] - t[3], t[5] - t[4], t[6] - t[5], t[7] - t[6], t[7] - t[0]);
  }
};

// A handful of requests on the default solver: one launch, arguments in, pinned memory out (tiny.cuh).  Returns whether
// it decided the batch.
bool TinySolve(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, const yd_task_req16* reqs16, uint32_t N, yd_grant* out,
               yd_grant8* out8, const yd_packed_ids& ids) {
  if ((!reqs && !reqs16) || N > yd::kTinyMax || s->solver_pref != 0 || !s->tiny_ok || s->sv.empty() || !s->n_comps) return false;
  s->h_small.ensure(256);
  yd::TinyArgs ta{};
  CopyRequests(reqs, reqs16, N, ta.reqs);
  ta.n = N; ta.now_ns = now_ns; ta.t = MakeTopo(s); ta.sv = s->arrays(); ta.ring = s->ring();
  ta.out = s->h_small.as<yd_grant>();
  ta.granted_out = reinterpret_cast<unsigned long long*>(s->h_small.as<char>() + yd::kTinyMax * sizeof(yd_grant));
  ta.counters = s->d_counters.as<Counters>();
  YD_CUDA_CHECK(cudaEventRecord(s->ev[0], s->st));
  yd::k_solve_tiny<<<1, 1024, 0, s->st>>>(ta);
  YD_CUDA_CHECK(cudaGetLastError());
  YD_CUDA_CHECK(cudaEventRecord(s->ev[5], s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
  WriteGrants(out, out8, ids, ta.out, N);
  const unsigned long long granted = *ta.granted_out;
  s->next_id += granted;
  s->staged_n = 0;
  float ms = 0;
  cudaEventElapsedTime(&ms, s->ev[0], s->ev[5]);
  ResetStats(s);
  yd_solve_stats& stt = s->stats;
  stt.total_ms = stt.solve_ms = ms;
  stt.decisions = N; stt.granted = granted; stt.kernel_launches = 1; stt.solver = 3;
  stt.h2d_bytes = 0;  // the requests are kernel arguments
  stt.d2h_bytes = size_t(N) * sizeof(yd_grant) + 8;  // written by the kernel into pinned host memory
  if (s->debug_env) {
    fprintf(stderr, "ydsched: solve n %u tiny 1 solver 3 spec 0 ring_cap %llu ring_lo %llu solve_ms %.3f\n", N,
            (unsigned long long)s->ring_cap, (unsigned long long)s->lo, ms);
  }
  return true;
}

// The device address of a page-locked caller array (yd_alloc_host), or null: pageable, or not 16-byte aligned.
void* MappedAddress(const void* p) {
  if (!p || (reinterpret_cast<uintptr_t>(p) & 15u)) return nullptr;
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return at.type == cudaMemoryTypeHost ? at.devicePointer : nullptr;
}

// The variant of an attempt (SoloTables::Choose); `now` is set to the kept-table signature a solo variant runs on.
SolveVariant ChooseVariant(yd_sched* s, uint32_t Nb, const SolveGeometry& geo, uint32_t solver, bool want_static, KeptSig& now) {
  const uint32_t S = (uint32_t)s->sv.size();
  // The fused front kernel takes batches in the latency-bound regime whose (class, tile) count matrices one block
  // scans in a few rounds; it needs the kept slot order.  Solo = it also writes the grants (no coupled component
  // had requests last time; if one has now, the kernel raises flag 4 and the batch is replayed with kFused).
  const bool fused = s->fused_cfg && s->fused_grid && s->solver_pref == 0 && solver == 2 && want_static && S &&
                     s->n_comps && Nb <= s->fused_max_nb && size_t(s->cls_bound) * geo.n_rtiles <= 32768 &&
                     size_t(s->cls_bound) * geo.n_ltiles <= 32768;
  if (fused && s->solo.hint) {
    now = KeptSig{CleanSig{g_buf_generation, s->z_cls_off, s->z_bytes, s->res_words, s->d_zero.p, s->d_res.p},
                  s->topo_gen, s->cls_bound};
  }
  // speculative (fused.cuh): every block holds at most two request tiles (their classes and ranks stay in
  // registers), the lists' offsets fit in shared memory, and registry positions fit the member words below the slot's
  // index in its tile (classes.cuh: kMemberSlotShift)
  const bool spec_ok = FusedLoffWords(s, geo) != 0 && geo.n_rtiles <= 2 * s->fused_grid && S <= yd::kMemberPosMask;
  return s->solo.Choose(fused, now, spec_ok);
}

// A solo solve: ONE kernel whose per-call scalars are kernel parameters, launched directly, as a graph would add a
// parameter patch and a graph launch to the call.  Its arguments are built before the events, which bracket what the
// solve enqueues on `st`; the kernel leaves grant count and flags in the mapped host record.  Returns the launches.
uint32_t LaunchSolo(yd_sched* s, uint32_t Nb, const SolveGeometry& geo, const SolvePlan& plan, bool copied, uint32_t packed,
                    HostProf& hp) {
  cudaStream_t st = s->st;
  const yd::FusedArgs a = MakeFusedArgs(s, Nb, geo, plan, false, packed & 1u, packed & 2u);
  hp.Stamp(3);
  YD_CUDA_CHECK(cudaEventRecord(s->ev[1], st));
  if (plan.variant == kSolo) {
    // the solo kernel keeps the verdicts in registers: only the class-table keys behind res[] are initialised --
    // and not even those when the previous solo solve left the scratch clean (kSoloClean, kSoloSpec)
    YD_CUDA_CHECK(cudaMemsetAsync(s->d_res.as<uint32_t>() + s->res_words, 0xFF, yd::kClsTableSize * 8, st));
    YD_CUDA_CHECK(cudaMemsetAsync(static_cast<char*>(s->d_zero.p) + s->z_cls_off, 0, s->z_bytes - s->z_cls_off, st));
  }
  WaitUpload(s, st, copied, false);
  LaunchFusedKernel(s, a);
  YD_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
  hp.Stamp(4);
  YD_CUDA_CHECK(cudaGetLastError());
  return 1;
}

// A general solve through the graph of its size class (EnqueueSolve, captured on first use).  Returns its launches.
uint32_t LaunchGraphed(yd_sched* s, uint32_t Nb, size_t slot_b, const SolveGeometry& geo, const SolvePlan& plan, bool copied,
                       uint32_t packed, HostProf& hp) {
  cudaStream_t st = s->st;
  yd_sched::GraphKey key;
  key.Nb = Nb; key.S = (uint32_t)s->sv.size(); key.n_comps = s->n_comps; key.max_comp = s->max_comp_servants;
  key.cls_bound = s->cls_bound; key.solver = plan.solver; key.wide = s->wide; key.slot_b = slot_b;
  key.gen = g_buf_generation; key.topo_gen = s->topo_gen; key.ring_cap = s->ring_cap;
  key.merge_rounds = plan.merge_rounds; key.force_stream = plan.force_stream;
  key.order_static = (plan.solver == 2 && s->order_static) ? 1u : 0u;
  key.variant = plan.variant; key.packed = packed;
  yd_sched::GraphEntry* hit = nullptr;
  for (auto& g : s->graphs) if (g.key == key) { hit = &g; break; }
  if (!hit) {
    cudaGraph_t graph = nullptr;
    YD_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    uint32_t l = EnqueueSolve(s, Nb, geo, plan, false, copied, true, packed);
    YD_CUDA_CHECK(cudaStreamEndCapture(st, &graph));
    cudaGraphExec_t exec = nullptr;
    YD_CUDA_CHECK(cudaGraphInstantiate(&exec, graph, 0));
    YD_CUDA_CHECK(cudaGraphDestroy(graph));
    if (s->graphs.size() >= 16) {  // drop the oldest size class
      cudaGraphExecDestroy(s->graphs.front().exec);
      s->graphs.erase(s->graphs.begin());
    }
    s->graphs.push_back(yd_sched::GraphEntry{key, exec, l});
    hit = &s->graphs.back();
  }
  hp.Stamp(3);
  YD_CUDA_CHECK(cudaEventRecord(s->ev[1], st));
  YD_CUDA_CHECK(cudaGraphLaunch(hit->exec, st));
  YD_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
  hp.Stamp(4);
  return hit->launches;
}

// YDSCHED_FUSED_PROF: the fused kernel's phase stamps after an attempt of `variant` on a batch of N.
void PrintFusedProfile(yd_sched* s, SolveVariant variant, uint32_t N) {
  if (variant == kSoloSpec) {
    unsigned long long t[9];
    YD_CUDA_CHECK(cudaMemcpy(t, s->d_fused_prof.p, sizeof t, cudaMemcpyDeviceToHost));
    if (s->h_meta.as<uint32_t>()[1] == yd::kFlagSpecMiss) {  // (no phase B)
      fprintf(stderr, "ydsched: fused variant 4 (speculative) n %u ns: A %llu barrier %llu missed\n", N, t[1] - t[0], t[2] - t[1]);
    } else {
      fprintf(stderr, "ydsched: fused variant 4 (speculative) n %u ns: A %llu barrier %llu B %llu total %llu (+tail %lld)\n", N,
              t[1] - t[0], t[2] - t[1], t[7] - t[2], t[7] - t[0], (long long)(t[8] - t[7]));
    }
    // every block's stamps (fused.cuh: kProfBlockWords), for tools/dev/phase_prof.py
    const uint32_t G = s->fused_grid;
    std::vector<unsigned long long> b(size_t(G) * yd::kProfBlockWords);
    YD_CUDA_CHECK(cudaMemcpy(b.data(), s->d_fused_prof.as<unsigned long long>() + yd::kProfHead, b.size() * 8,
                             cudaMemcpyDeviceToHost));
    std::string line = "ydsched: fused blocks " + std::to_string(G) + " last_end " + std::to_string(t[8]) + " stamps";
    for (unsigned long long v : b) line += " " + std::to_string(v);
    fprintf(stderr, "%s\n", line.c_str());
  } else if (variant != kPipeline) {
    unsigned long long t[9];
    YD_CUDA_CHECK(cudaMemcpy(t, s->d_fused_prof.p, sizeof t, cudaMemcpyDeviceToHost));
    fprintf(stderr, "ydsched: fused variant %u n %u ns: P1 %llu E1 %llu P3 %llu E2 %llu P5 %llu B3 %llu P6 %llu total %llu (+report/clean %lld)\n",
            (unsigned)variant, N, t[1] - t[0], t[2] - t[1], t[3] - t[2], t[4] - t[3], t[5] - t[4], t[6] - t[5], t[7] - t[6],
            t[7] - t[0], (long long)(t[8] - t[7]));
  }
}

// A call's stand-downs so far; `spec`: the speculative variant 0 not tried, 1 decided the batch, 2 missed (replayed).
struct StandDowns { int grow = 0, merge = 0; uint32_t spec = 0; };
enum AttemptEnd { kDecided, kAgain, kHalves };

// After an attempt, by its flag (meta[1]).  A slot-stream attempt with a flag decided nothing (the stream solver and
// the final kernels all stood down): `plan` is set up for the next attempt, or the batch is decided in halves.
AttemptEnd StandDown(yd_sched* s, SolvePlan& plan, StandDowns& d) {
  const uint32_t* meta = s->h_meta.as<uint32_t>();
  const uint32_t flag = meta[1];
  if (plan.solver != 2 || s->sv.empty() || !s->n_comps || flag == 0) {
    if (plan.variant == kSoloSpec) d.spec = 1;
    return kDecided;
  }
  if (flag == yd::kFlagSpecMiss) {
    // the kept class table could not decide the batch: replay without speculation (which builds the table again)
    d.spec = 2;
  } else if (flag == 4) {
    // the solo kernel met a component it cannot decide: the general sequence, now and next time (SoloTables::Take)
  } else if (flag == 2 && d.grow++ < 3 && GrowClassBound(s, meta)) {
    // more lists than provisioned: go again with the grown class bound
  } else if (flag == 3 && d.merge < 2) {
    // the merge solver's boundary states had not settled after the rounds in the graph: more
    // rounds first, then the sequential solver for everything it would have decided
    if (d.merge == 0) plan.MoreMergeRounds(s->merge_max_chunks);
    else plan.force_stream = 2;
    ++d.merge;
  } else if (s->max_comp_servants > kRowscanMaxComponent) {
    return kHalves;
  } else {
    plan.solver = 1;
  }
  return kAgain;
}

// More classes than the class table holds AND a component beyond the row-scan solver's reach.  n sequential decisions
// are the first half's followed by the second half's: decide the batch as two consecutive halves (each with half the
// requests, hence -- eventually -- few enough classes).  The stats are the second half's, with decisions = N.
void SolveInHalves(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, const yd_task_req16* reqs16, uint32_t N,
                   yd_grant* out, yd_grant8* out8, const yd_packed_ids& ids, bool keep8) {
  if (N < 2) { fprintf(stderr, "ydsched: class table overflow on a single request\n"); abort(); }
  std::vector<yd_task_req> r(N);
  if (reqs || reqs16) CopyRequests(reqs, reqs16, N, r.data());
  else YD_CUDA_CHECK(cudaMemcpy(r.data(), s->d_reqs.p, size_t(N) * sizeof(yd_task_req), cudaMemcpyDeviceToHost));
  std::vector<yd_grant> g(N);
  const uint32_t h = N / 2;
  yd_wait_for_starting_new_tasks(s, now_ns, r.data(), h, g.data());
  yd_wait_for_starting_new_tasks(s, now_ns, r.data() + h, N - h, g.data() + h);
  if (keep8) UploadGrants8(s, ids, g.data(), N);
  else WriteGrants(out, out8, ids, g.data(), N);
  s->stats.decisions = N;
}

// The stats of a decided batch (of the last attempt).  The event arithmetic costs a driver call apiece: done when
// yd_last_solve_stats asks, the events stay valid until the next solve.
void RecordSolveStats(yd_sched* s, uint32_t N, uint32_t launches, const SolvePlan& plan, const yd_task_req* reqs,
                      const yd_task_req16* reqs16, const yd_grant8* out8) {
  ResetStats(s);
  yd_solve_stats& stt = s->stats;
  s->stats_times_pending = (s->use_graphs || IsSolo(plan.variant)) ? 2 : 1;  // (graphed or solo: one device interval)
  stt.decisions = N; stt.granted = s->h_counters.as<Counters>()->granted; stt.kernel_launches = launches; stt.solver = plan.solver;
  stt.h2d_bytes = (reqs ? size_t(N) * sizeof(yd_task_req) : reqs16 ? size_t(N) * sizeof(yd_task_req16) : 0) + sizeof(yd::DynParams);
  stt.d2h_bytes = size_t(N) * (out8 ? sizeof(yd_grant8) : sizeof(yd_grant)) + sizeof(Counters) + 32;
}

// YDSCHED_DEBUG: which path the solve took (the last attempt, after any stand-down): `final` 0 = the solo kernel wrote
// the grants, 1 = k_final_fused, 3 = k_final_count / k_final_scan / k_final_write; `spec` over all attempts; the lease
// ring (`ring_lo` = the first live id) as the solve found it
void PrintSolveLine(yd_sched* s, uint32_t N, uint32_t Nb, size_t slot_b, const SolvePlan& plan, uint32_t spec) {
  const Counters* c = s->h_counters.as<Counters>();
  const uint32_t nb = (Nb + 1023) / 1024;
  const bool have_work = !s->sv.empty() && s->n_comps;
  const uint32_t solver = plan.solver;
  const bool solo = IsSolo(plan.variant), graphed = !solo && s->use_graphs;
  const uint32_t final_path = (solo && have_work && solver == 2) ? 0u : (solver == 2 && have_work && nb <= 2048) ? 1u : 3u;
  const auto back = solver == 2 && have_work && !solo ? MergeBack(s) : std::pair<uint32_t, uint32_t>{0, 0};
  fprintf(stderr, "ydsched: solve n %u tiny 0 variant %u order_static %d wide %d Nb %u slot_b %zu cls_bound %u final %u "
          "emask %d max_comp %zu solver %u graph %d merge_rounds %llu merge_chunks %llu walks %llu windows %llu "
          "merge_back %u merge_back_n %u spec %u ring_cap %llu ring_lo %llu solve_ms %.3f\n",
          N, (unsigned)plan.variant, (int)(solver == 2 && s->order_static), (int)s->wide, Nb, slot_b, s->cls_bound, final_path,
          (int)s->emask_ok, (size_t)s->max_comp_servants, solver, (int)graphed, c->pad[0], c->pad[1], c->pad[2],
          c->pad[3], back.first, back.second, spec, (unsigned long long)s->ring_cap, (unsigned long long)s->lo, s->stats.solve_ms);
}

// The solve behind yd_wait_for_starting_new_tasks and its packed twin.  Requests: `reqs` (24-byte records), or `reqs16`
// (16-byte records), or neither = the first n staged requests (yd_stage_requests) are already in HBM.  Grants: `out`
// (16-byte records) or `out8` (8-byte records, ids = first_task_id + ordinal * stride of BatchIds, also to ids_out), or
// with `keep8` neither: the 8-byte records stay in d_out8 for a device-side consumer (the RPC window, rpcs.cuh).
void WaitImpl(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, const yd_task_req16* reqs16, size_t n, yd_grant* out,
              yd_grant8* out8, yd_packed_ids* ids_out, bool keep8 = false) {
  const yd_packed_ids ids = BatchIds(s);
  if (ids_out) *ids_out = ids;
  if (n == 0) return;
  HostProf hp{s->host_prof};
  hp.Stamp(0);
  if (!reqs && !reqs16 && n > s->staged_n) { fprintf(stderr, "ydsched: NULL request array and nothing staged\n"); abort(); }
  CheckBatchSize(n);
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const uint32_t N = (uint32_t)n;
  const uint32_t S = (uint32_t)s->sv.size();
  const uint32_t packed = (reqs16 ? 1u : 0u) | (out8 || keep8 ? 2u : 0u);
  s->SyncServantState();
  s->SyncFacts();
  s->SyncTopology();
  s->EnsureRing(N);
  if (TinySolve(s, now_ns, reqs, reqs16, N, out, out8, ids)) return;

  // Size classes: grids, scratch arrays and memsets are dimensioned for the next power of
  // two; kernels read the exact n from DynParams.
  const uint32_t Nb = (uint32_t)NextPow2(N, 1024);
  // The slot table: kept across solves (all running_tasks values of every servant) while it is small enough,
  // else rebuilt per solve and clamped to the batch size.
  const size_t static_bound = S ? s->static_bound_cache : 0;  // (kept by SyncFacts)
  const bool want_static = s->solver_pref != 1 && static_bound <= kStaticSlotLimit;
  size_t slot_bound = static_bound;
  if (!want_static) {
    slot_bound = 0;
    for (auto&& v : s->sv) slot_bound += size_t(std::min(std::min(v.nproc, v.max_tasks), N)) + 1;
  }
  if (slot_bound > 0x7ffffff0ull) { fprintf(stderr, "ydsched: slot table too large\n"); abort(); }
  const size_t slot_b = (size_t)NextPow2(std::max<size_t>(slot_bound, 1), 4096);
  if (!want_static) s->order_static = false;
  EnsureSolveBuffers(s, Nb, slot_b);
  if (reqs16) s->d_reqs16.ensure(size_t(Nb) * sizeof(yd_task_req16));
  if (out8 || keep8) s->d_out8.ensure(size_t(Nb) * sizeof(yd_grant8));

  // solver choice: 2 (slot streams) unless asked otherwise or a component is too big for it
  // (the slot-stream solver takes components of any size: its sequential fallback keeps running_tasks of a
  // component beyond kStreamMaxComponent servants in HBM instead of shared memory)
  // (the row-scan solver holds 8192 servants per component)
  SolvePlan plan{kPipeline, s->solver_pref == 1 && s->max_comp_servants <= kRowscanMaxComponent ? 1u : 2u,
                 s->cfg_merge_rounds, s->cfg_force_stream};

  s->fsc.dyn = SetDynParams(s, N, N, now_ns);

  uint32_t launches = 0;
  hp.Stamp(1);
  YD_CUDA_CHECK(cudaEventRecord(s->ev[0], st));
  // The request upload runs on its own stream so that the slot table and its sort (which
  // do not read the requests) overlap it; consumers wait on ev_h2d, recorded after the copy.
  // (Page-locked caller arrays -- yd_alloc_host -- are not copied at all when the fused kernel runs: its first phase
  // reads the requests over PCIe itself and, solo, its last phase writes the grants straight into the caller's array.
  // Staged requests are in HBM already.  Neither waits for the copy stream.)
  bool copied = false;
  const void* in_host = reqs ? static_cast<const void*>(reqs) : static_cast<const void*>(reqs16);
  void* const in_dev = MappedAddress(in_host);
  void* const out_dev = MappedAddress(out ? static_cast<void*>(out) : static_cast<void*>(out8));
  if (in_host) s->staged_n = 0;  // the staging area now holds this batch
  StandDowns downs;
  for (;;) {
    memset(s->h_meta.p, 0, 32);
    // every buffer the sequence touches exists BEFORE a capture (no allocation inside one), and the scratch layout the
    // kept signature below describes is fixed
    if (plan.solver == 2) PrepareStreamBuffers(s, Nb, slot_b);
    const SolveGeometry geo = MakeGeometry(s, Nb, slot_b);
    KeptSig now;
    plan.variant = ChooseVariant(s, Nb, geo, plan.solver, want_static, now);
    // (a staged solve -- no request array in this call -- leaves its grants in HBM and copies them afterwards, so that
    // the device-side events around it time the solve alone)
    const bool solo = IsSolo(plan.variant);
    const bool zc_in = plan.variant != kPipeline && in_dev, zc_out = solo && out_dev && in_host;
    hp.Stamp(2);
    if (!zc_in && in_host && !copied) {
      YD_CUDA_CHECK(cudaMemcpyAsync(reqs ? s->d_reqs.p : s->d_reqs16.p, in_host,
                                    size_t(N) * (reqs ? sizeof(yd_task_req) : sizeof(yd_task_req16)), cudaMemcpyHostToDevice, s->st_copy));
      YD_CUDA_CHECK(cudaEventRecord(s->ev_h2d, s->st_copy));
      copied = true;
    }
    s->fsc.zc_in = zc_in ? in_dev : nullptr;
    s->fsc.zc_out = zc_out ? out_dev : nullptr;
    s->fsc.seq += 1;
    s->fsc.kept_fp = s->solo.kept_fp;
    *s->h_fsc.as<yd::FusedScalars>() = s->fsc;
    s->h_fio->done_seq = 0;
    if (plan.solver == 2 && want_static && S && s->n_comps && (s->order_dirty || !s->order_static || s->order_slot_b != slot_b)) {
      launches += RebuildSlotOrder(s, slot_b);
    }
    if (solo) launches += LaunchSolo(s, Nb, geo, plan, copied, packed, hp);
    else if (s->use_graphs) launches += LaunchGraphed(s, Nb, slot_b, geo, plan, copied, packed, hp);
    else launches += EnqueueSolve(s, Nb, geo, plan, true, copied, false, packed);
    if (plan.solver == 1) { s->order_dirty = true; s->order_static = false; }  // the row-scan solver's table overwrote the kept one
    if (zc_out || keep8) {}  // the kernel wrote the grants into the caller's page-locked array, or they stay in HBM
    else if (out8) YD_CUDA_CHECK(cudaMemcpyAsync(out8, s->d_out8.p, size_t(N) * sizeof(yd_grant8), cudaMemcpyDeviceToHost, st));
    else YD_CUDA_CHECK(cudaMemcpyAsync(out, s->d_out.p, size_t(N) * sizeof(yd_grant), cudaMemcpyDeviceToHost, st));
    YD_CUDA_CHECK(cudaEventRecord(s->ev[5], st));
    hp.Stamp(5);
    YD_CUDA_CHECK(cudaStreamSynchronize(st));
    hp.Stamp(6);
    if (solo) {  // the solo kernel's report: flags and grant count (no copy follows its launch)
      if (s->h_fio->done_seq != s->fsc.seq) { fprintf(stderr, "ydsched: the fused kernel left no report\n"); abort(); }
      memcpy(s->h_meta.p, const_cast<const uint32_t*>(s->h_fio->meta), 32);
      s->h_counters.as<Counters>()->granted = s->h_fio->granted;
    }
    if (s->fused_prof) PrintFusedProfile(s, plan.variant, N);
    s->solo.Take(plan.variant, s->h_meta.as<uint32_t>(), now, s->h_fio->classes_fp);
    const AttemptEnd end = StandDown(s, plan, downs);
    if (end == kHalves) return SolveInHalves(s, now_ns, reqs, reqs16, N, out, out8, ids, keep8);
    if (end == kDecided) break;
  }
  s->next_id += s->h_counters.as<Counters>()->granted;
  RecordSolveStats(s, N, launches, plan, reqs, reqs16, out8);
  hp.Print();
  if (s->debug_env) PrintSolveLine(s, N, Nb, slot_b, plan, downs.spec);
}
}  // namespace
}  // extern "C++"

// `reqs` == NULL: the first n staged requests (yd_stage_requests) are already in HBM.
void yd_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n,
                                    yd_grant* out) {
  WaitImpl(s, now_ns, reqs, nullptr, n, out, nullptr, nullptr);
}

// The same decisions with 16-byte requests up and 8-byte grants down (ydsched.h: yd_task_req16, yd_grant8).
void yd_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs, size_t n,
                                           yd_grant8* out, yd_packed_ids* ids) {
  WaitImpl(s, now_ns, nullptr, reqs, n, nullptr, out, ids);
}

extern "C++" {
namespace {
// KeepTaskAlive's upload to d_ids, then k_keep_alive writing `ok` (n flags of type Flag, on the device).  With one length
// (`lens` == null) the ids go up as they are.  With a length per id, the ids, the lengths and each id's last-occurrence
// mark go up in one copy; if the lengths are all equal this is the one-length call.
template <typename Flag>
void KeepAlive(yd_sched* s, int64_t now_ns, const uint64_t* ids, const int64_t* lens, size_t n, int64_t new_expires_in_ns,
               Flag* ok) {
  if (lens && std::all_of(lens, lens + n, [&](int64_t x) { return x == lens[0]; })) {
    new_expires_in_ns = lens[0];
    lens = nullptr;
  }
  const long long* d_lens = nullptr;
  const uint8_t* d_last = nullptr;
  if (!lens) {
    s->d_ids.ensure(n * 8);
    YD_CUDA_CHECK(cudaMemcpyAsync(s->d_ids.p, ids, n * 8, cudaMemcpyHostToDevice, s->st));
  } else {
    const size_t bytes = n * 17;  // ids (u64) | lengths (i64) | last-occurrence marks (u8)
    s->h_small.ensure(bytes);
    char* h = s->h_small.as<char>();
    memcpy(h, ids, n * 8);
    memcpy(h + n * 8, lens, n * 8);
    uint8_t* last = reinterpret_cast<uint8_t*>(h + n * 16);
    std::unordered_set<uint64_t> seen;
    seen.reserve(n);
    for (size_t i = n; i-- > 0;) last[i] = seen.insert(ids[i]).second ? 1 : 0;
    s->d_ids.ensure(bytes);
    YD_CUDA_CHECK(cudaMemcpyAsync(s->d_ids.p, h, bytes, cudaMemcpyHostToDevice, s->st));
    d_lens = reinterpret_cast<const long long*>(s->d_ids.as<char>() + n * 8);
    d_last = reinterpret_cast<const uint8_t*>(s->d_ids.as<char>() + n * 16);
  }
  yd::k_keep_alive<<<(unsigned)((n + 255) / 256), 256, 0, s->st>>>(s->d_ids.as<unsigned long long>(), (uint32_t)n,
                                                                    (long long)now_ns, (long long)new_expires_in_ns,
                                                                    d_lens, d_last, s->ring(), ok);
  YD_CUDA_CHECK(cudaGetLastError());
}

void KeepAliveHandle(yd_sched* s, int64_t now_ns, const uint64_t* ids, const int64_t* lens, size_t n,
                     int64_t new_expires_in_ns, uint8_t* ok_out) {
  if (n == 0) return;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->d_ok.ensure(n);
  KeepAlive(s, now_ns, ids, lens, n, new_expires_in_ns, s->d_ok.as<uint8_t>());
  YD_CUDA_CHECK(cudaMemcpyAsync(ok_out, s->d_ok.p, n, cudaMemcpyDeviceToHost, s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
}
}  // namespace
}  // extern "C++"

// KeepTaskAlive x n, cc:142-165.
void yd_keep_task_alive(yd_sched* s, int64_t now_ns, const uint64_t* ids, size_t n, int64_t new_expires_in_ns,
                        uint8_t* ok_out) {
  KeepAliveHandle(s, now_ns, ids, nullptr, n, new_expires_in_ns, ok_out);
}

// KeepTaskAlive x n, each with its own lease length.
void yd_keep_tasks_alive(yd_sched* s, int64_t now_ns, const uint64_t* ids, const int64_t* new_expires_in_ns, size_t n,
                         uint8_t* ok_out) {
  KeepAliveHandle(s, now_ns, ids, new_expires_in_ns, n, 0, ok_out);
}

// FreeTask x n, cc:167-188.  Fire and forget: ordered on the solve stream.
void yd_free_tasks(yd_sched* s, const uint64_t* ids, size_t n) {
  if (n == 0) return;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->SyncServantState();
  s->d_ids.ensure(n * 8);
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_ids.p, ids, n * 8, cudaMemcpyHostToDevice, s->st));
  yd::k_free<<<(unsigned)((n + 255) / 256), 256, 0, s->st>>>(s->d_ids.as<unsigned long long>(), (uint32_t)n,
                                                              s->ring(), s->d_run.as<uint32_t>(),
                                                              s->d_counters.as<Counters>(), s->shard ? s->d_dec.as<uint32_t>() : nullptr);
  YD_CUDA_CHECK(cudaGetLastError());
  // `ids` may be pageable and reused by the caller: the copy above has already
  // staged it (pageable H2D returns after staging) or the memory is pinned and we
  // must wait for the DMA.
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
}

// OnExpirationTimer, cc:498-536.
void yd_on_expiration_timer(yd_sched* s, int64_t now_ns) {
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  s->SyncServantState();
  const uint32_t S_old = (uint32_t)s->sv.size();
  std::vector<uint32_t> remap;
  uint32_t kept = 0;
  bool any_expired = false;
  for (auto&& v : s->sv) any_expired |= v.expires_at < now_ns;
  if (any_expired) {
    remap.resize(S_old);
    std::vector<ServantHost> alive;
    alive.reserve(S_old);
    for (uint32_t i = 0; i != S_old; ++i) {
      if (s->sv[i].expires_at < now_ns) {
        remap[i] = kNone;
        s->running.erase(s->sv[i].observed);  // RunningTaskBookkeeper::DropServant, cc:510-511
      } else {
        remap[i] = kept++;
        alive.push_back(std::move(s->sv[i]));
      }
    }
    s->sv.swap(alive);
    s->loc2pos.clear();
    for (uint32_t i = 0; i != s->sv.size(); ++i) s->loc2pos.emplace(s->sv[i].observed, i);
    s->topo_dirty = s->facts_dirty = s->order_dirty = true;
    s->d_remap.ensure(size_t(S_old) * 4);
    YD_CUDA_CHECK(cudaMemcpyAsync(s->d_remap.p, remap.data(), size_t(S_old) * 4, cudaMemcpyHostToDevice, st));
  }
  // min_live = ~0 before the pass
  YD_CUDA_CHECK(cudaMemsetAsync(&s->d_counters.as<Counters>()->min_live, 0xFF, 8, st));
  if (s->next_id > s->lo) {
    uint64_t cnt = s->next_id - s->lo;
    yd::k_tick<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(
        s->ring(), (long long)now_ns, any_expired ? s->d_remap.as<uint32_t>() : nullptr,
        s->d_counters.as<Counters>());
    YD_CUDA_CHECK(cudaGetLastError());
  }
  if (any_expired) {
    s->d_run_tmp.ensure(std::max<size_t>(size_t(S_old) * 4, 4));
    s->d_ever_tmp.ensure(std::max<size_t>(size_t(S_old) * 8, 8));
    if (s->shard) s->d_dec_tmp.ensure(std::max<size_t>(size_t(S_old) * 4, 4));
    yd::k_compact_servants<<<(S_old + 255) / 256, 256, 0, st>>>(
        S_old, s->d_remap.as<uint32_t>(), s->d_run.as<uint32_t>(), s->d_ever.as<unsigned long long>(),
        s->d_run_tmp.as<uint32_t>(), s->d_ever_tmp.as<unsigned long long>(), s->shard ? s->d_dec.as<uint32_t>() : nullptr,
        s->shard ? s->d_dec_tmp.as<uint32_t>() : nullptr);
    YD_CUDA_CHECK(cudaGetLastError());
    std::swap(s->d_run, s->d_run_tmp);
    std::swap(s->d_ever, s->d_ever_tmp);
    if (s->shard) std::swap(s->d_dec, s->d_dec_tmp);
    s->S_dev = kept;
  }
  s->FetchCounters();  // also makes `remap` (pageable) safe to drop
  const Counters* c = s->h_counters.as<Counters>();
  s->zombies_ub = c->zombies;
  s->lo = (c->min_live == ~0ull) ? s->next_id : c->min_live;
}

// KeepServantAlive x n (cc:190-220): registry work only, the facts go up before the next solve.
void yd_keep_servants_alive(yd_sched* s, int64_t now_ns, const yd_servant* servants, const int64_t* expires_in_ns, size_t n) {
  for (size_t i = 0; i != n; ++i) yd_keep_servant_alive(s, now_ns, &servants[i], expires_in_ns[i]);
}

extern "C++" {
namespace {
// NotifyServantRunningTasks (cc:222-277) for heartbeats of DISTINCT known servants: one upload, one
// sweep + one check kernel, one synchronisation, whatever the number of servants or reported tasks.
// `idx` = the items of the caller's array handled here, `pos` their registry positions.
// A range-sharded group's call (d_flags != nullptr) leaves the verdicts on the device instead: `tag` (rank + 1) per
// permitted id, as u32 words at d_flags[item_at[i] ..] for item i, the pass's items in registry order from `base`.  It neither
// downloads nor synchronises: the caller does, once, after the exchange.
void NotifyDistinct(yd_sched* s, const yd_heartbeat_item* items, const std::vector<uint32_t>& idx,
                    const std::vector<uint32_t>& pos, std::vector<std::vector<uint8_t>>& permitted,
                    uint32_t* d_flags = nullptr, uint32_t tag = 0, size_t base = 0, std::vector<size_t>* item_at = nullptr) {
  const uint32_t m = (uint32_t)idx.size();
  std::vector<uint32_t> order(m);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return pos[a] < pos[b]; });
  size_t total = 0;
  for (uint32_t k = 0; k != m; ++k) {
    if (item_at) (*item_at)[idx[order[k]]] = base + total;
    total += items[idx[order[k]]].n_tasks;
  }
  if (total > 0xfffffff0ull) { fprintf(stderr, "ydsched: heartbeat batch reports too many tasks\n"); abort(); }
  const bool window = s->next_id > s->lo;
  if (!window || (total == 0 && s->zombies_ub == 0)) return;  // nothing can be permitted, nothing to sweep
  // staging layout: ids[total] (u64) | item_off[m + 1] | item_pos[m] | (device only) permitted[total]
  const size_t b_ids = total * 8, b_off = (size_t(m) + 1) * 4, b_pos = size_t(m) * 4;
  s->h_small.ensure(b_ids + b_off + b_pos + total + 64);
  char* hb = s->h_small.as<char>();
  unsigned long long* h_ids = reinterpret_cast<unsigned long long*>(hb);
  uint32_t* h_off = reinterpret_cast<uint32_t*>(hb + b_ids);
  uint32_t* h_pos = h_off + m + 1;
  uint8_t* h_ok = reinterpret_cast<uint8_t*>(hb + b_ids + b_off + b_pos);
  size_t at = 0;
  for (uint32_t k = 0; k != m; ++k) {
    const yd_heartbeat_item& it = items[idx[order[k]]];
    h_off[k] = (uint32_t)at;
    h_pos[k] = pos[order[k]];
    for (size_t i = 0; i != it.n_tasks; ++i) h_ids[at++] = it.tasks[i].task_grant_id;
  }
  h_off[m] = (uint32_t)at;
  cudaStream_t st = s->st;
  s->d_ids.ensure(b_ids + b_off + b_pos + 8);
  s->d_ok.ensure(std::max<size_t>(total, 1));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_ids.p, hb, b_ids + b_off + b_pos, cudaMemcpyHostToDevice, st));
  yd::NotifyBatch nb{};
  nb.ids = s->d_ids.as<unsigned long long>();
  nb.item_off = reinterpret_cast<const uint32_t*>(s->d_ids.as<char>() + b_ids);
  nb.item_pos = nb.item_off + m + 1;
  nb.n_items = m;
  if (s->zombies_ub) {
    const uint64_t cnt = s->next_id - s->lo;
    yd::k_notify_sweep<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(s->ring(), nb, s->d_run.as<uint32_t>(),
                                                                       s->d_counters.as<Counters>(),
                                                                       s->shard ? s->d_dec.as<uint32_t>() : nullptr);
    YD_CUDA_CHECK(cudaGetLastError());
  }
  if (d_flags) {
    if (total) {
      yd::k_notify_check<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(s->ring(), nb, (uint32_t)total, d_flags + base, tag);
      YD_CUDA_CHECK(cudaGetLastError());
    }
    return;
  }
  if (total) {
    yd::k_notify_check<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(s->ring(), nb, (uint32_t)total, s->d_ok.as<uint8_t>(),
                                                                        uint8_t(1));
    YD_CUDA_CHECK(cudaGetLastError());
    YD_CUDA_CHECK(cudaMemcpyAsync(h_ok, s->d_ok.p, total, cudaMemcpyDeviceToHost, st));
  }
  s->FetchCounters();  // the one synchronisation
  s->zombies_ub = s->h_counters.as<Counters>()->zombies;
  for (uint32_t k = 0; k != m; ++k) {
    std::vector<uint8_t>& p = permitted[idx[order[k]]];
    if (total) memcpy(p.data(), h_ok + h_off[k], p.size());
  }
}

// The items' registry positions (kNone: the servant itself expired, every id is unknown, cc:243-245) and the passes
// of NotifyDistinct, `pass(idx, pos)` each.  Heartbeats of different servants touch disjoint leases, so any number of
// them is one device pass.  A servant that appears twice must see its first heartbeat's sweep: the batch is cut there.
template <typename Pass>
std::vector<uint32_t> NotifyPasses(yd_sched* s, const yd_heartbeat_item* items, size_t n, Pass&& pass) {
  std::vector<uint32_t> idx, pos;
  std::unordered_map<uint32_t, char> seen;
  std::vector<uint32_t> item_pos(n, kNone);
  for (size_t i = 0; i != n; ++i) {
    auto it = s->loc2pos.find(items[i].servant_location ? items[i].servant_location : "");
    if (it == s->loc2pos.end()) continue;
    item_pos[i] = it->second;
    if (seen.count(it->second)) {
      pass(idx, pos);
      idx.clear(); pos.clear(); seen.clear();
    }
    seen.emplace(it->second, 1);
    idx.push_back((uint32_t)i);
    pos.push_back(it->second);
  }
  if (!idx.empty()) pass(idx, pos);
  return item_pos;
}

// The answer, in request order, and the bookkeeper's update.  verdict(i, t) of task t of item i: 0 unknown, 1 permitted
// and kept here, 2 permitted and kept by the rank of a range-sharded group that holds its lease.
template <typename Verdict>
size_t NotifyAnswer(yd_sched* s, const yd_heartbeat_item* items, size_t n, const std::vector<uint32_t>& item_pos,
                    Verdict&& verdict, uint64_t* unknown_out, size_t* unknown_counts) {
  size_t total = 0;
  for (size_t i = 0; i != n; ++i) {
    const yd_heartbeat_item& it = items[i];
    size_t k = 0;
    if (item_pos[i] == kNone) {
      for (size_t t = 0; t != it.n_tasks; ++t) unknown_out[total + k++] = it.tasks[t].task_grant_id;
    } else {
      std::vector<RunningRec> kept;
      for (size_t t = 0; t != it.n_tasks; ++t) {
        const int v = verdict(i, t);
        if (v == 0) {
          unknown_out[total + k++] = it.tasks[t].task_grant_id;
        } else if (v == 1) {
          kept.push_back(RunningRec{it.tasks[t].servant_task_id, it.tasks[t].task_grant_id,
                                    it.tasks[t].servant_location ? it.tasks[t].servant_location : "",
                                    it.tasks[t].task_digest ? it.tasks[t].task_digest : "", (uint32_t)t});
        }
      }
      // RunningTaskBookkeeper::SetServantRunningTasks, running_task_bookkeeper.cc:24-29
      s->running.erase(it.servant_location);
      s->running.emplace(it.servant_location, std::move(kept));
    }
    if (unknown_counts) unknown_counts[i] = k;
    total += k;
  }
  return total;
}
}  // namespace
}  // extern "C++"

// NotifyServantRunningTasks x n, in array order (cc:222-277).
size_t yd_notify_servants_running_tasks(yd_sched* s, const yd_heartbeat_item* items, size_t n, uint64_t* unknown_out,
                                        size_t* unknown_counts) {
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->SyncServantState();
  std::vector<std::vector<uint8_t>> permitted(n);
  for (size_t i = 0; i != n; ++i) permitted[i].assign(items[i].n_tasks, 0);
  const std::vector<uint32_t> item_pos = NotifyPasses(
      s, items, n, [&](const std::vector<uint32_t>& idx, const std::vector<uint32_t>& pos) { NotifyDistinct(s, items, idx, pos, permitted); });
  return NotifyAnswer(
      s, items, n, item_pos, [&](size_t i, size_t t) { return permitted[i][t] ? 1 : 0; }, unknown_out, unknown_counts);
}

// NotifyServantRunningTasks, cc:222-277: a batch of one.
size_t yd_notify_servant_running_tasks(yd_sched* s, const char* servant_location, const yd_running_task* tasks,
                                       size_t n, uint64_t* unknown_out) {
  const yd_heartbeat_item item{servant_location, tasks, n};
  return yd_notify_servants_running_tasks(s, &item, 1, unknown_out, nullptr);
}

// RunningTaskBookkeeper::GetRunningTasks, running_task_bookkeeper.cc:36-43.
size_t yd_get_running_tasks(yd_sched* s, yd_running_task* out, size_t cap) {
  s->running_cache.clear();
  for (auto&& [k, v] : s->running) s->running_cache.insert(s->running_cache.begin(), v.begin(), v.end());
  for (size_t i = 0; i < s->running_cache.size() && i < cap; ++i) {
    auto&& t = s->running_cache[i];
    out[i] = yd_running_task{t.servant_task_id, t.task_grant_id, t.servant_location.c_str(), t.task_digest.c_str()};
  }
  return s->running_cache.size();
}

size_t yd_num_servants(yd_sched* s) { return s->sv.size(); }

uint64_t yd_grant_capacity_bound(yd_sched* s) {
  uint64_t b = 0;
  for (auto&& v : s->sv) b += std::min(v.nproc, v.max_tasks);
  return b;
}

const char* yd_servant_location(yd_sched* s, uint32_t idx) {
  return idx < s->sv.size() ? s->sv[idx].observed.c_str() : nullptr;
}

size_t yd_get_servant_state(yd_sched* s, yd_servant_state* out, size_t cap) {
  const size_t S = s->sv.size();
  if (!S || !cap) return S;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->SyncServantState();
  std::vector<uint32_t> run(S);
  std::vector<unsigned long long> ever(S);
  YD_CUDA_CHECK(cudaMemcpyAsync(run.data(), s->d_run.p, S * 4, cudaMemcpyDeviceToHost, s->st));
  YD_CUDA_CHECK(cudaMemcpyAsync(ever.data(), s->d_ever.p, S * 8, cudaMemcpyDeviceToHost, s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
  for (size_t i = 0; i < S && i < cap; ++i) {
    const ServantHost& v = s->sv[i];
    uint64_t capav = (s->FactFlags(v) & yd::kFlagLowMem)
                         ? run[i]
                         : (uint64_t)yd::capacity_at(v.max_tasks, v.nproc, v.load, run[i]);
    out[i] = yd_servant_state{run[i], ever[i], capav, v.expires_at};
  }
  return S;
}

int yd_get_servant_personality(yd_sched* s, uint32_t idx, yd_servant* out) {
  if (idx >= s->sv.size()) return 0;
  const ServantHost& v = s->sv[idx];
  s->personality_envs.clear();
  for (uint32_t e : v.envs) s->personality_envs.push_back(s->envs[e].c_str());
  if (out) {
    *out = yd_servant{v.version, v.priority, v.reason, (uint32_t)v.envs.size(), v.observed.c_str(), v.reported.c_str(),
                      s->personality_envs.data(), v.nproc, v.load, v.max_tasks, 0, v.total_mem, v.avail_mem};
  }
  return 1;
}

uint64_t yd_next_task_id(yd_sched* s) { return BatchIds(s).first_task_id; }

uint64_t yd_num_tasks(yd_sched* s) {
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->FetchCounters();
  return s->h_counters.as<Counters>()->alive;
}

int yd_last_solve_stats(yd_sched* s, yd_solve_stats* out) {
  if (!s->have_stats) return 0;
  if (s->stats_times_pending) {
    float ms = 0;
    yd_solve_stats& stt = s->stats;
    cudaEventElapsedTime(&ms, s->ev[0], s->ev[5]); stt.total_ms = ms;
    if (s->stats_times_pending == 2) {
      // inside a graph, or around the one solo launch, the phases are not separable: solve_ms is the whole device pipeline
      cudaEventElapsedTime(&ms, s->ev[1], s->ev[4]); stt.solve_ms = ms;
    } else {
      cudaEventElapsedTime(&ms, s->ev[1], s->ev[2]); stt.prep_ms = ms;
      cudaEventElapsedTime(&ms, s->ev[2], s->ev[3]); stt.solve_ms = ms;
      cudaEventElapsedTime(&ms, s->ev[3], s->ev[4]); stt.final_ms = ms;
    }
    s->stats_times_pending = 0;
  }
  *out = s->stats;
  return 1;
}

void* yd_alloc_host(size_t bytes) {
  void* p = nullptr;
  // Mapped + portable up to 32 MB: the fused kernel reads requests from / writes grants to such arrays directly (batches
  // up to 262 144 requests).  Bigger arrays only ever go through the copy engines and are allocated as before (plain
  // page-locked memory: the 240 MB + 160 MB arrays of a 10 M-request batch copied at 16 GB/s when mapped, 45 GB/s when not).
  const unsigned flags = bytes <= (32u << 20) ? (cudaHostAllocMapped | cudaHostAllocPortable) : cudaHostAllocDefault;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, flags) != cudaSuccess) return nullptr;
  return p;
}
void yd_free_host(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
#include "ydsched_rpc_impl.inc"
#include "yddump_impl.inc"
#include "ydservice_impl.inc"
#include "ydwire_impl.inc"

// ---- a window of WaitForStartingTask RPCs decided on the device (include/ydrpcs_packed.h, rpcs.cuh) -----------------
extern "C" {
// The range-sharded group's part of a window (shard_host.inc).
static std::vector<unsigned long long> ShardRanges(const yd_sched* s, size_t total, size_t* lo, size_t* hi);
static int ShardDecideWindow(yd_sched* s, int64_t now_ns, const std::vector<unsigned long long>& counts);
}  // extern "C"

extern "C++" {
namespace {
bool ShardRefusesWide(yd_sched* s);  // (shard_host.inc)

// Windows of at most this many decisions keep the host expansion: on the host their queue goes to the one-launch tiny
// solve (k_solve_tiny, the requests as kernel arguments), which a staged queue cannot take, so expanding on the device
// would trade that one launch for an upload, six launches and the general solve.
constexpr size_t kHostWindowMax = yd::kTinyMax;

// yd_wait_for_starting_task_rpcs_packed, and with `group` its range-sharded form.  The host computes the window's size
// and its refusals (O(n_rpcs), nothing per decision) and uploads the RPC records; the device expands the window into the
// staged queue (this handle's range of it), the staged solve decides it with its 8-byte grants left in HBM (on a group:
// gathered from every rank, device to device), and the report writes the results and the grants in ordinal order.
size_t RpcWindow(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs, yd_rpc_wait_result* results,
                 yd_grant8* grants_out, size_t cap, yd_packed_ids* ids, bool group) {
  const yd_packed_ids id0 = BatchIds(s);  // (a group's next_id is replicated)
  if (ids) *ids = id0;
  const size_t total = yd_rpc_expanded_requests(s, rpcs, n_rpcs);
  if (!yd_rpc_detail::Fits(total, cap)) return (size_t)-1;
  if (total == 0 || (!group && total <= kHostWindowMax) || n_rpcs >= 0x40000000ull) {
    // the definition itself: the unpacked call, the grants packed
    static thread_local yd_rpc_detail::HostStage stage;
    yd_grant* g = static_cast<yd_grant*>(stage.ensure(std::max<size_t>(total, 1) * sizeof(yd_grant)));
    if (!g) return (size_t)-1;
    const size_t k = group ? yd_shard_wait_for_starting_task_rpcs(s, now_ns, rpcs, n_rpcs, results, g, cap)
                           : yd_wait_for_starting_task_rpcs(s, now_ns, rpcs, n_rpcs, results, g, cap);
    if (k != (size_t)-1) WriteGrants(nullptr, grants_out, id0, g, k);
    return k;
  }
  if (group && ShardRefusesWide(s)) return (size_t)-1;  // (before anything changes, as the unpacked group call refuses)
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const uint64_t bound = yd_grant_capacity_bound(s);
  const uint32_t n = (uint32_t)n_rpcs, T = (uint32_t)total;
  // this handle's range [lo, hi) of the queue: all of it, or a group rank's (ShardRanges)
  size_t lo = 0, hi = total;
  std::vector<unsigned long long> counts;
  if (group) counts = ShardRanges(s, total, &lo, &hi);
  s->d_rpcs.ensure(n_rpcs * sizeof(yd_rpc_wait));
  s->d_rpc_off.ensure((n_rpcs + 1) * 4);
  s->d_rpc_ng.ensure((n_rpcs + 1) * 4);
  s->d_rpc_res.ensure(n_rpcs * sizeof(yd_rpc_wait_result));
  s->d_rpc_out.ensure(total * sizeof(yd_grant8));
  s->d_out8.ensure(total * sizeof(yd_grant8));  // (a group's gathered window)
  // the staged queue at its size class, so that the solve does not reallocate it
  s->d_reqs.ensure(size_t(NextPow2(std::max<size_t>(hi - lo, 1), 1024)) * sizeof(yd_task_req));
  const yd_rpc_wait* d_rpcs = s->d_rpcs.as<yd_rpc_wait>();
  uint32_t* off = s->d_rpc_off.as<uint32_t>();
  uint32_t* ng = s->d_rpc_ng.as<uint32_t>();
  yd_rpc_wait_result* res = s->d_rpc_res.as<yd_rpc_wait_result>();
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rpcs.p, rpcs, n_rpcs * sizeof(yd_rpc_wait), cudaMemcpyHostToDevice, st));
  yd::k_rpc_count<<<(n + 255) / 256, 256, 0, st>>>(d_rpcs, n, bound, off);
  yd::k_scan_u32<<<1, 1024, 0, st>>>(off, n + 1, nullptr, 0, nullptr, 0);
  uint32_t launches = 2;
  if (hi > lo) {
    yd::k_rpc_expand<<<(unsigned)((hi - lo + 255) / 256), 256, 0, st>>>(d_rpcs, n, bound, off, (uint32_t)lo, (uint32_t)hi,
                                                                        s->d_reqs.as<yd_task_req>());
    launches += 1;
  }
  YD_CUDA_CHECK(cudaGetLastError());
  // the solve reads the staged queue on `st`, after the expansion
  s->staged_n = hi - lo;
  const uint64_t next0 = s->next_id;
  if (group) {
    if (ShardDecideWindow(s, now_ns, counts)) return (size_t)-1;
  } else {
    WaitImpl(s, now_ns, nullptr, nullptr, total, nullptr, nullptr, nullptr, true);
  }
  s->staged_n = 0;  // as the unpacked call leaves it: its queue went through the staging area
  const uint64_t granted = s->next_id - next0;
  const uint2* g8 = s->d_out8.as<uint2>();
  yd::k_rpc_grants<<<(n + 255) / 256, 256, 0, st>>>(d_rpcs, n, off, g8, ng, res);
  yd::k_scan_u32<<<1, 1024, 0, st>>>(ng, n + 1, nullptr, 0, nullptr, 0);
  yd::k_rpc_report<<<(std::max(n, T) + 255) / 256, 256, 0, st>>>(n, T, off, g8, ng, res, s->d_rpc_out.as<uint2>());
  launches += 3;
  YD_CUDA_CHECK(cudaGetLastError());
  YD_CUDA_CHECK(cudaMemcpyAsync(results, res, n_rpcs * sizeof(yd_rpc_wait_result), cudaMemcpyDeviceToHost, st));
  if (granted) YD_CUDA_CHECK(cudaMemcpyAsync(grants_out, s->d_rpc_out.p, granted * sizeof(yd_grant8), cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  for (size_t i = 0; i != n_rpcs; ++i) {
    if (results[i].reserved) {
      fprintf(stderr, "ydsched: RPC %zu of a window has a grant outside its leading run\n", i);
      abort();
    }
  }
  if (!group) {
    // the solve's stats, as the window's: its decisions, the kernels around the solve, and the window's records moved
    // (the solve's scalars -- DynParams up, the counters down -- are not counted)
    yd_solve_stats& stt = s->stats;
    stt.decisions = total;
    stt.kernel_launches += launches;
    stt.h2d_bytes = n_rpcs * sizeof(yd_rpc_wait);
    stt.d2h_bytes = n_rpcs * sizeof(yd_rpc_wait_result) + granted * sizeof(yd_grant8);
  }
  if (s->debug_env) {
    fprintf(stderr, "ydsched: rpcs n_rpcs %zu decisions %zu range %zu %zu granted %llu expanded on device\n", n_rpcs, total,
            lo, hi, (unsigned long long)granted);
  }
  return granted;
}
}  // namespace
}  // extern "C++"

size_t yd_wait_for_starting_task_rpcs_packed(yd_sched* s, int64_t now_ns, const yd_rpc_wait* rpcs, size_t n_rpcs,
                                             yd_rpc_wait_result* results, yd_grant8* grants_out, size_t cap,
                                             yd_packed_ids* ids) {
  return RpcWindow(s, now_ns, rpcs, n_rpcs, results, grants_out, cap, ids, false);
}

// ---- compilation-cache bloom pre-filter (bloom.cuh) ------------------------------------------
extern "C" {

int yd_bloom_reset(yd_sched* s, uint64_t size_in_bits, uint32_t num_hashes) {
  if (size_in_bits == 0 || size_in_bits > (1ull << 30) || num_hashes == 0) return 1;
  uint64_t bits = 8;  // max(8, next_pow2(m)) (bloom_filter.h:214-219)
  while (bits < size_in_bits) bits <<= 1;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  const size_t alloc = std::max<size_t>(bits / 8, 4);  // the kernels address the table as le32 words
  s->d_bloom.ensure(alloc);
  YD_CUDA_CHECK(cudaMemsetAsync(s->d_bloom.p, 0, alloc, s->st));
  s->bloom_bits = bits;
  s->bloom_hashes = num_hashes;
  return 0;
}

int yd_bloom_load(yd_sched* s, const uint8_t* bytes, size_t n_bytes, uint32_t num_hashes) {
  if (n_bytes == 0 || ((n_bytes * 8) & (n_bytes * 8 - 1)) || num_hashes == 0) return 1;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  s->d_bloom.ensure(std::max<size_t>(n_bytes, 4));
  YD_CUDA_CHECK(cudaMemsetAsync(s->d_bloom.p, 0, 4, s->st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_bloom.p, bytes, n_bytes, cudaMemcpyHostToDevice, s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
  s->bloom_bits = n_bytes * 8;
  s->bloom_hashes = num_hashes;
  return 0;
}

static void BloomRun(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride, uint8_t* out) {
  if (!s->bloom_bits) { fprintf(stderr, "ydsched: bloom filter used before yd_bloom_reset / yd_bloom_load\n"); abort(); }
  if (key_len > yd::kBloomMaxKey) { fprintf(stderr, "ydsched: bloom keys longer than %d bytes\n", yd::kBloomMaxKey); abort(); }
  if (n == 0) return;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  const size_t span = (n - 1) * stride + key_len;
  s->d_bloom_keys.ensure(span ? span : 1);
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_bloom_keys.p, keys, span, cudaMemcpyHostToDevice, s->st));
  const unsigned grid = (unsigned)((n + 127) / 128);
  const yd::BloomRecords recs{s->d_bloom_keys.as<unsigned char>(), stride, (uint32_t)key_len};
  if (out) {
    s->d_bloom_out.ensure(n);
    yd::k_bloom<false><<<grid, 128, 0, s->st>>>(recs, (uint32_t)n, s->bloom_hashes, s->bloom_bits - 1,
                                                s->d_bloom.as<uint32_t>(), s->d_bloom_out.as<uint8_t>());
    YD_CUDA_CHECK(cudaGetLastError());
    YD_CUDA_CHECK(cudaMemcpyAsync(out, s->d_bloom_out.p, n, cudaMemcpyDeviceToHost, s->st));
  } else {
    yd::k_bloom<true><<<grid, 128, 0, s->st>>>(recs, (uint32_t)n, s->bloom_hashes, s->bloom_bits - 1,
                                               s->d_bloom.as<uint32_t>(), nullptr);
    YD_CUDA_CHECK(cudaGetLastError());
  }
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
}

void yd_bloom_add(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride) {
  BloomRun(s, keys, n, key_len, stride, nullptr);
}

void yd_bloom_possibly_contains(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride, uint8_t* out) {
  if (!out) return;
  BloomRun(s, keys, n, key_len, stride, out);
}

size_t yd_bloom_get_bytes(yd_sched* s, uint8_t* out, size_t cap) {
  const size_t nbytes = s->bloom_bits / 8;
  if (out && cap && nbytes) {
    YD_CUDA_CHECK(cudaSetDevice(s->device));
    YD_CUDA_CHECK(cudaMemcpyAsync(out, s->d_bloom.p, std::min(cap, nbytes), cudaMemcpyDeviceToHost, s->st));
    YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
  }
  return nbytes;
}

// ---- in-flight task index (running_index.cuh) ---------------------------------------------------

static yd::RtIndex MakeRtIndex(yd_sched* s) {
  yd::RtIndex ix{};
  ix.bytes = s->d_rt_bytes.as<unsigned char>();
  ix.off = s->d_rt_off.as<uint32_t>();
  ix.len = s->d_rt_len.as<uint32_t>();
  ix.slots = s->rt_snapshot.empty() ? nullptr : s->d_rt_slots.as<uint32_t>();
  ix.mask = s->rt_mask;
  return ix;
}

// The index over s->rt_snapshot (running_index.cuh).  Returns the number of entries.
static size_t RtIndexBuild(yd_sched* s) {
  const size_t n = s->rt_snapshot.size();
  s->rt_distinct = 0;
  if (n == 0) return 0;
  if (n > 0x7fffffffull) { fprintf(stderr, "ydsched: running-task snapshot too large\n"); abort(); }
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  // digests packed on 8-byte boundaries so the kernels can use word loads
  std::vector<uint32_t> off(n), len(n);
  std::vector<unsigned long long> ids(n);
  size_t total = 0;
  for (size_t i = 0; i < n; ++i) {
    off[i] = (uint32_t)total;
    len[i] = (uint32_t)s->rt_snapshot[i].task_digest.size();
    ids[i] = s->rt_snapshot[i].servant_task_id;
    total += (len[i] + 7) & ~size_t(7);
    if (total > 0xfffffff0ull) { fprintf(stderr, "ydsched: running-task digests exceed 4 GiB\n"); abort(); }
  }
  std::vector<unsigned char> bytes(total ? total : 8, 0);
  for (size_t i = 0; i < n; ++i) memcpy(bytes.data() + off[i], s->rt_snapshot[i].task_digest.data(), len[i]);
  uint64_t cap = 1024;
  while (cap < 2 * n) cap <<= 1;  // load factor <= 0.5
  s->rt_mask = (uint32_t)(cap - 1);
  s->d_rt_bytes.ensure(bytes.size());
  s->d_rt_off.ensure(n * 4);
  s->d_rt_len.ensure(n * 4);
  s->d_rt_ids.ensure(n * 8);
  s->d_rt_slots.ensure(cap * 4 + 4);  // + the distinct-digest counter
  cudaStream_t st = s->st;
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_bytes.p, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_off.p, off.data(), n * 4, cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_len.p, len.data(), n * 4, cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_ids.p, ids.data(), n * 8, cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaMemsetAsync(s->d_rt_slots.p, 0, cap * 4 + 4, st));
  uint32_t* distinct = s->d_rt_slots.as<uint32_t>() + cap;
  yd::k_rt_build<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(MakeRtIndex(s), (uint32_t)n, distinct);
  YD_CUDA_CHECK(cudaGetLastError());
  uint32_t h_distinct = 0;
  YD_CUDA_CHECK(cudaMemcpyAsync(&h_distinct, distinct, 4, cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));  // also keeps the pageable staging vectors alive long enough
  s->rt_distinct = h_distinct;
  return n;
}

// RunningTaskKeeper::Refresh, running_task_keeper.cc:40-65.
size_t yd_running_index_refresh(yd_sched* s) {
  // the snapshot: what GetRunningTasks answers now (running_task_bookkeeper.cc:36-43)
  // (each servant's list goes to the FRONT there: same order, built back to front in O(n))
  s->rt_snapshot.clear();
  {
    std::vector<const std::vector<RunningRec>*> groups;
    for (auto&& [k, v] : s->running) groups.push_back(&v);
    for (auto it = groups.rbegin(); it != groups.rend(); ++it) {
      s->rt_snapshot.insert(s->rt_snapshot.end(), (*it)->begin(), (*it)->end());
    }
  }
  return RtIndexBuild(s);
}

size_t yd_running_index_size(yd_sched* s) { return s->rt_distinct; }

// RunningTaskKeeper::TryFindTask x n, running_task_keeper.cc:67-75.
void yd_running_index_find(yd_sched* s, const char* keys, size_t n, size_t key_len, size_t stride,
                           yd_running_hit* out) {
  if (n == 0 || !out) return;
  if (n > 0x7fffffffull || key_len > 0x7fffffffull) { fprintf(stderr, "ydsched: running-index query too large\n"); abort(); }
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const size_t span = (n - 1) * stride + key_len;
  s->d_rt_keys.ensure(span ? span : 1);
  s->d_rt_out.ensure(n * sizeof(yd_running_hit));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_keys.p, keys, span, cudaMemcpyHostToDevice, st));
  yd::k_rt_find<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      MakeRtIndex(s), yd::RtRecords{s->d_rt_keys.as<unsigned char>(), stride, (uint32_t)key_len}, (uint32_t)n,
      s->d_rt_ids.as<unsigned long long>(), s->d_rt_out.as<uint4>());
  YD_CUDA_CHECK(cudaGetLastError());
  YD_CUDA_CHECK(cudaMemcpyAsync(out, s->d_rt_out.p, n * sizeof(yd_running_hit), cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
}

int yd_running_index_entry(yd_sched* s, uint32_t i, yd_running_task* out) {
  if (i >= s->rt_snapshot.size()) return 0;
  auto&& t = s->rt_snapshot[i];
  if (out) *out = yd_running_task{t.servant_task_id, t.task_grant_id, t.servant_location.c_str(), t.task_digest.c_str()};
  return 1;
}

// The pre-filtered solve's buffers for a queue of N requests, cache keys (key_span bytes) if `bloom`, task digests
// (digest_span bytes) if `dedupe`.  Drops the staged queue.
static void FilterPrepare(yd_sched* s, uint32_t N, bool bloom, size_t key_span, bool dedupe, size_t digest_span) {
  const uint32_t nt = (N + 1023) / 1024;
  s->d_freqs.ensure(size_t(N) * sizeof(yd_task_req));
  s->d_fverdict.ensure(N);
  s->d_ftile.ensure(size_t(nt + 1) * 4);
  s->d_reqs.ensure(size_t(NextPow2(N, 1024)) * sizeof(yd_task_req));
  s->h_fcount.ensure(16);
  s->staged_n = 0;
  if (bloom) {
    s->d_bloom_keys.ensure(key_span ? key_span : 1);
    s->d_bloom_out.ensure(N);
  }
  if (dedupe) {
    s->d_rt_keys.ensure(digest_span ? digest_span : 1);
    s->d_rt_out.ensure(size_t(N) * sizeof(yd_running_hit));
  }
}

// The pre-filters' keys on the device (d_bloom_keys, d_rt_keys): fixed-length records of len bytes at a stride
// (yd_prefilter), or with `binary` contiguous 32-byte digests (yd_prefilter_packed).
struct FilterKeys {
  bool bloom = false, dedupe = false, binary = false;
  size_t key_len = 0, key_stride = 0, digest_len = 0, digest_stride = 0;
};

// The compaction: the offered requests of d_freqs (24-byte records, or with `req16` 16-byte ones) -> the solver's queue.
static void KeepScatter(yd_sched* s, uint32_t N, bool req16) {
  if (req16) {
    yd::keep_scatter(s->d_freqs.as<yd_task_req16>(), s->d_fverdict.as<uint8_t>(), s->d_ftile.as<uint32_t>(), N,
                     s->d_reqs.as<yd_task_req>(), s->st);
  } else {
    yd::keep_scatter(s->d_freqs.as<yd_task_req>(), s->d_fverdict.as<uint8_t>(), s->d_ftile.as<uint32_t>(), N,
                     s->d_reqs.as<yd_task_req>(), s->st);
  }
}

// The last step of the pre-filtered solve on a rank of a range-sharded group (shard_host.inc).
static size_t ShardSolveKept(yd_sched* s, int64_t now_ns, uint32_t N, uint32_t kept, bool req16, yd_grant* grants_out,
                             yd_grant8* out8, yd_packed_ids* ids);

// The device part of the pre-filtered solve, from the first filter stage on: the queue is in d_freqs (16-byte records if
// `req16`), the keys `k` in d_bloom_keys / d_rt_keys, and ev_f[0] has been recorded.  The solve of the compacted queue is
// the single handle's, or with `group` the range-sharded group's; its grants go to grants_out, or packed with *ids to
// out8.
static size_t FilterStages(yd_sched* s, int64_t now_ns, uint32_t N, const FilterKeys& k, bool req16, uint8_t* verdict_out,
                           yd_running_hit* hits_out, yd_grant* grants_out, yd_grant8* out8, yd_packed_ids* ids,
                           size_t h2d_bytes, uint32_t extra_launches, bool group) {
  cudaStream_t st = s->st;
  const size_t n = N;
  const uint32_t nt = (N + 1023) / 1024;
  if (k.bloom) {
    unsigned char* keys = s->d_bloom_keys.as<unsigned char>();
    if (k.binary) {
      yd::k_bloom<false><<<(N + 127) / 128, 128, 0, st>>>(yd::BloomCacheDigests{keys}, N, s->bloom_hashes, s->bloom_bits - 1,
                                                          s->d_bloom.as<uint32_t>(), s->d_bloom_out.as<uint8_t>());
    } else {
      yd::k_bloom<false><<<(N + 127) / 128, 128, 0, st>>>(yd::BloomRecords{keys, k.key_stride, (uint32_t)k.key_len}, N,
                                                          s->bloom_hashes, s->bloom_bits - 1, s->d_bloom.as<uint32_t>(),
                                                          s->d_bloom_out.as<uint8_t>());
    }
  }
  if (k.dedupe) {
    unsigned char* keys = s->d_rt_keys.as<unsigned char>();
    if (k.binary) {
      yd::k_rt_find<<<(N + 255) / 256, 256, 0, st>>>(MakeRtIndex(s), yd::RtTaskDigests{keys}, N,
                                                     s->d_rt_ids.as<unsigned long long>(), s->d_rt_out.as<uint4>());
    } else {
      yd::k_rt_find<<<(N + 255) / 256, 256, 0, st>>>(MakeRtIndex(s), yd::RtRecords{keys, k.digest_stride, (uint32_t)k.digest_len},
                                                     N, s->d_rt_ids.as<unsigned long long>(), s->d_rt_out.as<uint4>());
    }
  }
  yd::keep_count_scan(k.bloom ? s->d_bloom_out.as<uint8_t>() : nullptr, k.dedupe ? s->d_rt_out.as<uint4>() : nullptr, N,
                      s->d_fverdict.as<uint8_t>(), s->d_ftile.as<uint32_t>(), st);
  KeepScatter(s, N, req16);
  YD_CUDA_CHECK(cudaGetLastError());
  YD_CUDA_CHECK(cudaEventRecord(s->ev_f[1], st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->h_fcount.p, s->d_ftile.as<uint32_t>() + nt, 4, cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaMemcpyAsync(verdict_out, s->d_fverdict.p, N, cudaMemcpyDeviceToHost, st));
  if (hits_out) {
    if (k.dedupe) YD_CUDA_CHECK(cudaMemcpyAsync(hits_out, s->d_rt_out.p, n * sizeof(yd_running_hit), cudaMemcpyDeviceToHost, st));
    else for (size_t i = 0; i != n; ++i) hits_out[i] = yd_running_hit{0, YD_NO_SERVANT, 0};
  }
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  const uint32_t kept = *s->h_fcount.as<uint32_t>();
  float filter_ms = 0;
  cudaEventElapsedTime(&filter_ms, s->ev_f[0], s->ev_f[1]);
  size_t ret = kept;
  if (group) {
    ret = ShardSolveKept(s, now_ns, N, kept, req16, grants_out, out8, ids);
    s->stats.total_ms = filter_ms;
  } else if (kept) {
    s->staged_n = kept;  // the compaction wrote the solver's queue
    WaitImpl(s, now_ns, nullptr, nullptr, kept, grants_out, out8, ids);
    yd_solve_stats st2;
    yd_last_solve_stats(s, &st2);  // (turns the solve's events into milliseconds before they are reused)
  } else {
    if (ids) *ids = BatchIds(s);
    ResetStats(s);
  }
  // stats of the whole call: prep = the filter stages + compaction (device), solve / final = the solve's, decisions = n
  s->stats.prep_ms += filter_ms;
  s->stats.decisions = N;
  s->stats.kernel_launches += 3 + (k.bloom ? 1 : 0) + (k.dedupe ? 1 : 0) + extra_launches;
  s->stats.h2d_bytes += h2d_bytes;
  s->stats.d2h_bytes += N + 4 + (hits_out && k.dedupe ? n * sizeof(yd_running_hit) : 0);
  return ret;
}

// BASELINE configs[3] in one call: bloom probes, in-flight index probes, order-preserving compaction and the solve,
// with the queue resident in HBM from the first stage to the last (filter.cuh).  The requests are `reqs` (24-byte records)
// with the keys of `f`, and the grants 16-byte records in grants_out; or, packed, `reqs16` (16-byte records) with the
// digests of `fp`, and the grants 8-byte records in out8 with *ids.  `group`: the solve is the range-sharded group's
// (yd_shard_filter_and_wait_for_starting_new_tasks and its packed twin).
static size_t FilterCall(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, const yd_task_req16* reqs16, size_t n,
                         const yd_prefilter* f, const yd_prefilter_packed* fp, uint8_t* verdict_out, yd_running_hit* hits_out,
                         yd_grant* grants_out, yd_grant8* out8, yd_packed_ids* ids, bool group) {
  if (n == 0) {
    if (group) return ShardSolveKept(s, now_ns, 0, 0, false, grants_out, out8, ids);
    if (ids) *ids = BatchIds(s);
    return 0;
  }
  CheckBatchSize(n);
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const uint32_t N = (uint32_t)n;
  const bool req16 = reqs16 != nullptr;
  FilterKeys k;
  const void *key_src = nullptr, *digest_src = nullptr;
  if (fp) {
    k.binary = true;
    k.bloom = fp->cache_digests, k.dedupe = fp->task_digests;
    key_src = fp->cache_digests, digest_src = fp->task_digests;
  } else if (f) {
    k.bloom = f->cache_keys, k.dedupe = f->task_digests;
    key_src = f->cache_keys, digest_src = f->task_digests;
    k.key_len = f->cache_key_len, k.key_stride = f->cache_key_stride;
    k.digest_len = f->task_digest_len, k.digest_stride = f->task_digest_stride;
  }
  if (k.bloom) {
    if (!s->bloom_bits) { fprintf(stderr, "ydsched: bloom filter used before yd_bloom_reset / yd_bloom_load\n"); abort(); }
    if (k.key_len > yd::kBloomMaxKey) { fprintf(stderr, "ydsched: bloom keys longer than %d bytes\n", yd::kBloomMaxKey); abort(); }
  }
  const size_t key_span = !k.bloom ? 0 : k.binary ? n * 32 : (n - 1) * k.key_stride + k.key_len;
  const size_t digest_span = !k.dedupe ? 0 : k.binary ? n * 32 : (n - 1) * k.digest_stride + k.digest_len;
  const size_t req_bytes = size_t(N) * (req16 ? sizeof(yd_task_req16) : sizeof(yd_task_req));
  FilterPrepare(s, N, k.bloom, key_span, k.dedupe, digest_span);
  // uploads: the queue, the cache keys, the task digests (one stream: each stage starts when its input has landed)
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_freqs.p, req16 ? static_cast<const void*>(reqs16) : reqs, req_bytes,
                                cudaMemcpyHostToDevice, st));
  if (k.bloom) YD_CUDA_CHECK(cudaMemcpyAsync(s->d_bloom_keys.p, key_src, key_span, cudaMemcpyHostToDevice, st));
  if (k.dedupe) YD_CUDA_CHECK(cudaMemcpyAsync(s->d_rt_keys.p, digest_src, digest_span, cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaEventRecord(s->ev_f[0], st));
  return FilterStages(s, now_ns, N, k, req16, verdict_out, hits_out, grants_out, out8, ids, req_bytes + key_span + digest_span,
                      0, group);
}

size_t yd_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n,
                                                 const yd_prefilter* f, uint8_t* verdict_out, yd_running_hit* hits_out,
                                                 yd_grant* grants_out) {
  return FilterCall(s, now_ns, reqs, nullptr, n, f, nullptr, verdict_out, hits_out, grants_out, nullptr, nullptr, false);
}

size_t yd_filter_and_wait_for_starting_new_tasks_packed(yd_sched* s, int64_t now_ns, const yd_task_req16* reqs, size_t n,
                                                        const yd_prefilter_packed* filter, uint8_t* verdict_out,
                                                        yd_running_hit* hits_out, yd_grant8* grants_out,
                                                        yd_packed_ids* ids) {
  return FilterCall(s, now_ns, nullptr, reqs, n, nullptr, filter, verdict_out, hits_out, nullptr, grants_out, ids, false);
}

// ---- cache keys and task digests from task descriptors (blake3.cuh) ------------------------------------------------

// Appends the digests interned since the last derivation to the device env table (yd_intern_env, heartbeats and
// yd_import_state all intern through `envs`, which only grows).  Returns the bytes uploaded.
static size_t SyncEnvTable(yd_sched* s) {
  const size_t E = s->envs.size();
  if (E == s->env_dev_n && s->d_env_off) return 0;
  cudaStream_t st = s->st;
  std::vector<uint32_t> off(E - s->env_dev_n + 1);
  std::string bytes;
  off[0] = (uint32_t)s->env_dev_bytes;
  for (size_t e = s->env_dev_n; e != E; ++e) {
    bytes += s->envs[e];
    if (s->env_dev_bytes + bytes.size() > 0xffffff00ull) { fprintf(stderr, "ydsched: interned digests exceed 4 GiB\n"); abort(); }
    off[e - s->env_dev_n + 1] = (uint32_t)(s->env_dev_bytes + bytes.size());
  }
  // grown by doubling, stream-ordered; the old contents are copied over
  auto grow = [&](auto*& p, size_t used, size_t need, size_t& cap) {
    if (need <= cap && p) return;
    size_t ncap = std::max<size_t>(std::max(need, cap * 2), 256);
    void* np = nullptr;
    YD_CUDA_CHECK(cudaMallocAsync(&np, ncap + 8, st));  // + 8: LoadU32 reads whole aligned words
    if (p) {
      if (used) YD_CUDA_CHECK(cudaMemcpyAsync(np, p, used, cudaMemcpyDeviceToDevice, st));
      YD_CUDA_CHECK(cudaFreeAsync(p, st));
    }
    p = static_cast<std::remove_reference_t<decltype(p)>>(np);
    cap = ncap;
  };
  grow(s->d_env_bytes, s->env_dev_bytes, s->env_dev_bytes + bytes.size(), s->env_cap_bytes);
  grow(s->d_env_off, (s->env_dev_n + 1) * 4, (E + 1) * 4, s->env_cap_n);
  if (!bytes.empty())
    YD_CUDA_CHECK(cudaMemcpyAsync(s->d_env_bytes + s->env_dev_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_env_off + s->env_dev_n, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));  // (the staging strings go out of scope)
  s->env_dev_n = E;
  s->env_dev_bytes += bytes.size();
  return bytes.size() + off.size() * 4;
}

// The per-call descriptors on the device, in one stream-ordered scratch allocation (StateTmp's discipline: the
// grow-only buffers, whose reallocation drops the kept class table, are not touched).  `reqs_dev` is where the kernel
// reads the requests' env ids; null: they are uploaded into the scratch too.
struct KeyScratch {
  void* base = nullptr;
  size_t h2d = 0;
  yd::KeySources ks{};
};

static KeyScratch UploadKeySources(yd_sched* s, const yd_task_req* reqs, const yd_task_req* reqs_dev, size_t n,
                                   const yd_task_sources* src, size_t out_bytes) {
  cudaStream_t st = s->st;
  KeyScratch k;
  k.h2d = SyncEnvTable(s);
  auto al = [](size_t b) { return (b + 15) & ~size_t(15); };
  const size_t args_b = src->args_offsets[src->n_args], off_b = (src->n_args + 1) * 8, idx_b = n * 4;
  const size_t sd_b = src->source_digest_len ? (n - 1) * src->source_digest_stride + src->source_digest_len : 0;
  const size_t req_b = reqs_dev ? 0 : n * sizeof(yd_task_req);
  const size_t total = al(args_b + 8) + al(off_b) + al(idx_b) + al(sd_b + 8) + al(req_b) + out_bytes;
  YD_CUDA_CHECK(cudaMallocAsync(&k.base, total, st));
  char* p = static_cast<char*>(k.base);
  auto put = [&](const void* h, size_t b, size_t room) {
    if (b) YD_CUDA_CHECK(cudaMemcpyAsync(p, h, b, cudaMemcpyHostToDevice, st));
    k.h2d += b;
    char* at = p;
    p += al(room);
    return at;
  };
  k.ks.args = reinterpret_cast<const unsigned char*>(put(src->args, args_b, args_b + 8));
  k.ks.args_off = reinterpret_cast<const unsigned long long*>(put(src->args_offsets, off_b, off_b));
  k.ks.args_index = reinterpret_cast<const uint32_t*>(put(src->args_index, idx_b, idx_b));
  k.ks.src = reinterpret_cast<const unsigned char*>(put(src->source_digests, sd_b, sd_b + 8));
  k.ks.reqs = reqs_dev ? reqs_dev : reinterpret_cast<const yd_task_req*>(put(reqs, req_b, req_b));
  k.ks.src_stride = src->source_digest_stride;
  k.ks.src_len = (uint32_t)src->source_digest_len;
  k.ks.env_bytes = s->d_env_bytes;
  k.ks.env_off = s->d_env_off;
  k.ks.n = (uint32_t)n;
  k.ks.cache_keys = reinterpret_cast<unsigned char*>(p);  // the outputs' room, if any (the caller points them elsewhere)
  return k;
}

static void LaunchTaskKeys(yd_sched* s, yd::KeySources ks) {
  ks.both = ks.cache_keys && ks.task_digests;
  const size_t threads = size_t(ks.n) << ks.both;
  yd::k_task_keys<<<(unsigned)((threads + 127) / 128), 128, 0, s->st>>>(ks);
  YD_CUDA_CHECK(cudaGetLastError());
}

int yd_derive_task_keys(yd_sched* s, const yd_task_req* reqs, size_t n, const yd_task_sources* src, char* cache_keys_out,
                        char* task_digests_out) {
  if (int rc = yd_keys_check(s->envs, reqs, n, src)) return rc;
  if (n == 0 || (!cache_keys_out && !task_digests_out)) return YD_KEYS_OK;
  CheckBatchSize(n);
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const size_t kb = cache_keys_out ? n * YD_KEYS_CACHE_KEY_LEN : 0, db = task_digests_out ? n * YD_KEYS_TASK_DIGEST_LEN : 0;
  KeyScratch k = UploadKeySources(s, reqs, nullptr, n, src, kb + db);
  unsigned char* room = k.ks.cache_keys;
  k.ks.cache_keys = cache_keys_out ? room : nullptr;
  k.ks.task_digests = task_digests_out ? room + kb : nullptr;
  LaunchTaskKeys(s, k.ks);
  if (cache_keys_out) YD_CUDA_CHECK(cudaMemcpyAsync(cache_keys_out, room, kb, cudaMemcpyDeviceToHost, st));
  if (task_digests_out) YD_CUDA_CHECK(cudaMemcpyAsync(task_digests_out, room + kb, db, cudaMemcpyDeviceToHost, st));
  YD_CUDA_CHECK(cudaFreeAsync(k.base, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  return YD_KEYS_OK;
}

// The pre-filtered solve from descriptors: the keys are derived straight into d_bloom_keys / d_rt_keys, at the strides
// the filter stages read, so from there on it is yd_filter_and_wait_for_starting_new_tasks' device part unchanged.  The
// descriptors have passed yd_keys_check.  `group`: the solve is the range-sharded group's.
static size_t DeriveFilterCall(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n, const yd_task_sources* src,
                               uint32_t stages, uint8_t* verdict_out, yd_running_hit* hits_out, yd_grant* grants_out,
                               bool group) {
  if (n == 0) return group ? ShardSolveKept(s, now_ns, 0, 0, false, grants_out, nullptr, nullptr) : 0;
  CheckBatchSize(n);
  const bool bloom = stages & YD_STAGE_CACHE, dedupe = stages & YD_STAGE_DEDUPE;
  if (bloom && !s->bloom_bits) { fprintf(stderr, "ydsched: bloom filter used before yd_bloom_reset / yd_bloom_load\n"); abort(); }
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  const uint32_t N = (uint32_t)n;
  FilterPrepare(s, N, bloom, n * YD_KEYS_CACHE_KEY_LEN, dedupe, n * YD_KEYS_TASK_DIGEST_LEN);
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_freqs.p, reqs, size_t(N) * sizeof(yd_task_req), cudaMemcpyHostToDevice, st));
  KeyScratch k{};
  if (bloom || dedupe) {
    k = UploadKeySources(s, reqs, s->d_freqs.as<yd_task_req>(), n, src, 0);
    k.ks.cache_keys = bloom ? s->d_bloom_keys.as<unsigned char>() : nullptr;
    k.ks.task_digests = dedupe ? s->d_rt_keys.as<unsigned char>() : nullptr;
  }
  YD_CUDA_CHECK(cudaEventRecord(s->ev_f[0], st));  // (prep_ms: from the derivation on)
  if (bloom || dedupe) {
    LaunchTaskKeys(s, k.ks);
    YD_CUDA_CHECK(cudaFreeAsync(k.base, st));
  }
  FilterKeys fk;
  fk.bloom = bloom, fk.dedupe = dedupe;
  fk.key_len = fk.key_stride = YD_KEYS_CACHE_KEY_LEN;
  fk.digest_len = fk.digest_stride = YD_KEYS_TASK_DIGEST_LEN;
  return FilterStages(s, now_ns, N, fk, false, verdict_out, hits_out, grants_out, nullptr, nullptr,
                      size_t(N) * sizeof(yd_task_req) + k.h2d, (bloom || dedupe) ? 1u : 0u, group);
}

size_t yd_derive_filter_and_wait_for_starting_new_tasks(yd_sched* s, int64_t now_ns, const yd_task_req* reqs, size_t n,
                                                        const yd_task_sources* src, uint32_t stages, uint8_t* verdict_out,
                                                        yd_running_hit* hits_out, yd_grant* grants_out) {
  if (yd_keys_check(s->envs, reqs, n, src) != YD_KEYS_OK) return (size_t)-1;
  return DeriveFilterCall(s, now_ns, reqs, n, src, stages, verdict_out, hits_out, grants_out, false);
}


}  // extern "C"

// ---- state export / import (include/ydstate.h): host side; the lease passes are in state.cuh ----------------------
namespace {

bool IsFresh(const yd_sched* s) {
  return s->sv.empty() && s->next_id == 0 && s->lo == 0 && s->running.empty() && s->running.bucket_count() == 1 &&
         s->envs.empty() && s->ips.size() == 1 && s->staged_n == 0;
}

// Stream-ordered temporaries (cudaMallocAsync): the export's and the import's scratch never enters a captured graph, so
// it stays out of the grow-only buffers whose reallocation bumps g_buf_generation -- that bump would drop the captured
// graphs and the kept class table, i.e. cost the next solve its speculation.
void* StateTmp(yd_sched* s, size_t bytes) {
  void* p = nullptr;
  YD_CUDA_CHECK(cudaMallocAsync(&p, std::max<size_t>(bytes, 8), s->st));
  return p;
}

}  // namespace

namespace {

// The live leases of the ring's window: per 1024-id block a count, scanned (k_state_count + k_final_scan).  `n` is
// valid after the stream's next synchronisation; the scratch goes with FreeLiveLeases.
struct LiveLeases {
  uint32_t nb = 0;
  uint32_t* d_off = nullptr;
  Counters* d_sum = nullptr;
  unsigned long long n = 0;
};

void CountLiveLeases(yd_sched* s, LiveLeases* L) {
  cudaStream_t st = s->st;
  L->nb = (uint32_t)((s->next_id - s->lo + 1023) / 1024);
  if (!L->nb) return;
  char* t = static_cast<char*>(StateTmp(s, sizeof(Counters) + size_t(L->nb) * 4));
  L->d_sum = reinterpret_cast<Counters*>(t);
  L->d_off = reinterpret_cast<uint32_t*>(t + sizeof(Counters));
  YD_CUDA_CHECK(cudaMemsetAsync(L->d_sum, 0, sizeof(Counters), st));
  yd::k_state_count<<<L->nb, 1024, 0, st>>>(s->ring(), L->d_off);
  YD_CUDA_CHECK(cudaGetLastError());
  // the exclusive scan of the grant path, into a scratch Counters (its total lands in ->granted)
  yd::k_final_scan<<<1, 1024, 0, st>>>(L->d_off, L->nb, L->d_sum, nullptr);
  YD_CUDA_CHECK(cudaGetLastError());
  YD_CUDA_CHECK(cudaMemcpyAsync(&L->n, &L->d_sum->granted, 8, cudaMemcpyDeviceToHost, st));
}

// The counted leases as records, in id order, at d_rec.
void WriteLiveLeases(yd_sched* s, const LiveLeases& L, int64_t now_ns, yd::StateLease* d_rec) {
  yd::k_state_write<<<L.nb, 1024, 0, s->st>>>(s->ring(), (long long)now_ns, L.d_off, d_rec);
  YD_CUDA_CHECK(cudaGetLastError());
}

void FreeLiveLeases(yd_sched* s, const LiveLeases& L) {
  if (L.d_sum) YD_CUDA_CHECK(cudaFreeAsync(L.d_sum, s->st));
}

// Every section of the export but the lease records (n_leases stays 0).  Synchronises the stream.
ydstate::StateImage HostImage(yd_sched* s, int64_t now_ns) {
  const size_t S = s->sv.size();
  std::vector<unsigned long long> ever(S);
  if (S) YD_CUDA_CHECK(cudaMemcpyAsync(ever.data(), s->d_ever.p, S * 8, cudaMemcpyDeviceToHost, s->st));
  YD_CUDA_CHECK(cudaStreamSynchronize(s->st));
  ydstate::StateImage im;
  im.id_stride = s->id_stride;
  im.id_offset = s->id_offset;
  im.min_mem = s->min_mem;
  im.next_task_id = yd_next_task_id(s);
  im.envs = s->envs;
  im.ips = s->ips;
  im.servants.resize(S);
  for (size_t i = 0; i != S; ++i) {
    const ServantHost& v = s->sv[i];
    ydstate::Servant& o = im.servants[i];
    o.version = v.version; o.priority = v.priority; o.reason = v.reason;
    o.nproc = v.nproc; o.load = v.load; o.max_tasks = v.max_tasks;
    o.total_mem = v.total_mem; o.avail_mem = v.avail_mem;
    o.expires_rel = v.expires_at - now_ns;
    o.ever = ever[i];
    o.observed = v.observed; o.reported = v.reported;
    o.envs.reserve(v.envs.size());
    for (uint32_t e : v.envs) o.envs.push_back(s->envs[e]);
  }
  im.bucket_count = s->running.bucket_count();
  for (auto&& [loc, v] : s->running) {
    ydstate::Group& g = im.groups.emplace_back();
    g.location = loc;
    for (auto&& t : v) g.tasks.push_back(ydstate::Task{t.servant_task_id, t.task_grant_id, t.servant_location, t.task_digest});
  }
  return im;
}

// The leases [*k0, *k1) (ascending id order) that rank `rank` of `world` holds after an import: lease k of n goes to
// rank k * world / n, contiguous id blocks.  One rank holds all of them.
void HeldBlock(uint64_t n, uint32_t rank, uint32_t world, uint64_t* k0, uint64_t* k1) {
  *k0 = (uint64_t(rank) * n + world - 1) / world;
  *k1 = (uint64_t(rank + 1) * n + world - 1) / world;
}

uint32_t LeaseHolder(const ydstate::StateImage& im, uint64_t task_grant_id, uint32_t world) {
  const auto& L = im.leases;
  auto it = std::lower_bound(L.begin(), L.end(), task_grant_id, [](const ydstate::Lease& l, uint64_t id) { return l.id < id; });
  if (it == L.end() || it->id != task_grant_id) return 0;  // a bookkeeper entry whose lease is gone: rank 0 keeps it
  return (uint32_t)(uint64_t(it - L.begin()) * world / L.size());
}

// Everything an import can refuse, checked before anything changes: freshness, the blob, the config, and room on the
// device for the ring of the leases this rank will hold.
int CheckImport(yd_sched* s, const uint8_t* blob, size_t len, uint32_t rank, uint32_t world, ydstate::StateImage* im) {
  if (!IsFresh(s)) return YD_STATE_NOT_FRESH;
  if (int rc = ydstate::DecodeState(blob, len, im)) return rc;
  if (im->id_stride != s->id_stride || im->id_offset != s->id_offset || im->min_mem != s->min_mem) return YD_STATE_CONFIG_MISMATCH;
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  auto local = [&](uint64_t ext) { return (ext - im->id_offset) / im->id_stride; };
  uint64_t k0, k1;
  HeldBlock(im->leases.size(), rank, world, &k0, &k1);
  const uint64_t next_id = local(im->next_task_id);
  const uint64_t lo = k0 < k1 ? local(im->leases[k0].id) : next_id;
  // The ring is sized from the oldest live id, as EnsureRing would have grown it (DecodeState bounds the window by
  // kMaxWindow, so none of this overflows); a valid export that cannot fit the device's free memory now is refused.
  uint64_t ring_cap = 1ull << 16;
  while (ring_cap < (next_id - lo) * 2) ring_cap <<= 1;
  size_t free_b = 0, total_b = 0;
  YD_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
  if (ring_cap * 16 + im->leases.size() * sizeof(yd::StateLease) > free_b) return YD_STATE_NO_MEMORY;
  return YD_STATE_OK;
}

// Loads a checked image: the replicated state in full, the leases rank `rank` of `world` holds into the ring, every
// lease into running_tasks, and the bookkeeper entries whose lease the rank holds.
void ApplyImport(yd_sched* s, int64_t now_ns, const ydstate::StateImage& im, uint32_t rank, uint32_t world) {
  cudaStream_t st = s->st;
  auto local = [&](uint64_t ext) { return (ext - im.id_offset) / im.id_stride; };
  const size_t n = im.leases.size();
  uint64_t k0, k1;
  HeldBlock(n, rank, world, &k0, &k1);
  const uint64_t next_id = local(im.next_task_id);
  const uint64_t lo = k0 < k1 ? local(im.leases[k0].id) : next_id;

  // host side: exactly what KeepServantAlive, the interning calls and the bookkeeper would have built
  s->envs = im.envs;
  s->ips = im.ips;
  s->env_ids.clear();
  s->ip_ids.clear();
  for (uint32_t i = 0; i != s->envs.size(); ++i) s->env_ids.emplace(s->envs[i], i);
  for (uint32_t i = 0; i != s->ips.size(); ++i) s->ip_ids.emplace(s->ips[i], i);
  const uint32_t S = (uint32_t)im.servants.size();
  std::vector<unsigned long long> ever(S);
  for (uint32_t i = 0; i != S; ++i) {
    const ydstate::Servant& v = im.servants[i];
    ServantHost& rec = s->sv.emplace_back();
    rec.version = v.version; rec.priority = v.priority; rec.reason = v.reason;
    rec.observed = v.observed; rec.reported = v.reported;
    for (auto&& e : v.envs) rec.envs.push_back(s->InternEnv(e));
    rec.nproc = v.nproc; rec.load = v.load; rec.max_tasks = v.max_tasks;
    rec.total_mem = v.total_mem; rec.avail_mem = v.avail_mem;
    rec.discovered_at = now_ns;
    rec.expires_at = now_ns + v.expires_rel;
    s->loc2pos.emplace(rec.observed, i);
    ever[i] = v.ever;
  }
  // the bookkeeper's iteration order: same bucket count, groups inserted last-first (ydstate.h); every rank has every
  // group, as every rank sees every heartbeat
  if (im.bucket_count != 1) s->running.rehash(im.bucket_count);
  for (auto g = im.groups.rbegin(); g != im.groups.rend(); ++g) {
    std::vector<RunningRec> v;
    for (uint32_t j = 0; j != g->tasks.size(); ++j) {
      const ydstate::Task& t = g->tasks[j];
      if (world == 1 || LeaseHolder(im, t.task_grant_id, world) == rank)
        v.push_back(RunningRec{t.servant_task_id, t.task_grant_id, t.servant_location, t.task_digest, j});
    }
    s->running.emplace(g->location, std::move(v));
  }
  s->topo_dirty = s->facts_dirty = s->order_dirty = true;  // the first solve rebuilds topology, facts and slot order

  // device side: servant state, the ring, the counters
  if (S) {
    s->d_run.ensure(size_t(S) * 4);
    s->d_ever.ensure(size_t(S) * 8);
    YD_CUDA_CHECK(cudaMemsetAsync(s->d_run.p, 0, size_t(S) * 4, st));
    YD_CUDA_CHECK(cudaMemcpyAsync(s->d_ever.p, ever.data(), size_t(S) * 8, cudaMemcpyHostToDevice, st));
    if (s->shard) {  // every rank's running_tasks is the whole group's: nothing to hand to the others
      s->d_dec.ensure(size_t(S) * 4);
      YD_CUDA_CHECK(cudaMemsetAsync(s->d_dec.p, 0, size_t(S) * 4, st));
    }
  }
  s->S_dev = S;
  s->d_t_exp.release(); s->d_t_srv.release(); s->d_t_flags.release();
  s->ring_cap = 0;
  s->lo = lo;
  s->next_id = next_id;
  s->EnsureRing(0);
  uint64_t zombies = 0;
  for (uint64_t k = k0; k < k1; ++k) zombies += (im.leases[k].flags & YD_STATE_LEASE_ZOMBIE) != 0;
  if (n) {
    yd::StateLease* d_rec = static_cast<yd::StateLease*>(StateTmp(s, n * sizeof(yd::StateLease)));
    YD_CUDA_CHECK(cudaMemcpyAsync(d_rec, im.leases.data(), n * sizeof(yd::StateLease), cudaMemcpyHostToDevice, st));
    yd::k_state_scatter<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_rec, (uint32_t)n, (uint32_t)k0, (uint32_t)k1, s->ring(),
                                                                    (long long)now_ns, s->d_run.as<uint32_t>());
    YD_CUDA_CHECK(cudaGetLastError());
    YD_CUDA_CHECK(cudaFreeAsync(d_rec, st));
  }
  Counters* c = s->h_counters.as<Counters>();
  memset(c, 0, sizeof(Counters));
  c->alive = k1 - k0;
  c->zombies = zombies;
  c->min_live = ~0ull;
  YD_CUDA_CHECK(cudaMemcpyAsync(s->d_counters.p, c, sizeof(Counters), cudaMemcpyHostToDevice, st));
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  s->zombies_ub = zombies;
}

}  // namespace

extern "C" size_t yd_export_state(yd_sched* s, int64_t now_ns, uint8_t* out, size_t cap) {
  if (s->shard) return 0;  // a range-sharded handle holds part of the leases: yd_shard_export_state
  YD_CUDA_CHECK(cudaSetDevice(s->device));
  cudaStream_t st = s->st;
  s->SyncServantState();
  LiveLeases L;
  CountLiveLeases(s, &L);
  ydstate::StateImage im = HostImage(s, now_ns);
  im.n_leases = L.n;  // (written straight into `out` below)
  size_t lease_off = 0;
  const size_t size = ydstate::EncodeState(im, out, cap, &lease_off);
  if (out && cap >= size && L.n) {
    yd::StateLease* d_rec = static_cast<yd::StateLease*>(StateTmp(s, L.n * sizeof(yd::StateLease)));
    WriteLiveLeases(s, L, now_ns, d_rec);
    YD_CUDA_CHECK(cudaMemcpyAsync(out + lease_off, d_rec, L.n * sizeof(yd::StateLease), cudaMemcpyDeviceToHost, st));
    YD_CUDA_CHECK(cudaFreeAsync(d_rec, st));
  }
  FreeLiveLeases(s, L);
  YD_CUDA_CHECK(cudaStreamSynchronize(st));
  return size;
}

extern "C" int yd_import_state(yd_sched* s, int64_t now_ns, const uint8_t* blob, size_t len) {
  if (s->shard) return YD_STATE_UNSUPPORTED;  // yd_shard_import_state
  ydstate::StateImage im;
  if (int rc = CheckImport(s, blob, len, 0, 1, &im)) return rc;
  ApplyImport(s, now_ns, im, 0, 1);
  return YD_STATE_OK;
}

// ---- range-sharded queue over the GPUs of a node (include/ydshard.h) ------------------------------------
#include "shard_host.inc"
#include "shard_calls.inc"
