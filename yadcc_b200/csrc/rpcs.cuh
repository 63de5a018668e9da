// rpcs.cuh -- a window of WaitForStartingTask RPCs (yd_wait_for_starting_task_rpcs_packed, include/ydrpcs_packed.h)
// expanded into the solver's queue and reported on the device: 32 bytes per RPC go up, the staged solve decides the
// queue in HBM, 16 bytes per RPC and 8 per grant come back.  The rules are include/ydsched_rpc_impl.inc's (Expand,
// FillRange, Report), restated per RPC and per decision.
//
//   k_rpc_count    decisions per RPC: ClampReqs(immediate) + ClampReqs(prefetch), 0 for an INVALID_ARGUMENT RPC
//   (k_scan_u32    exclusive scan: where each RPC's decisions start, the window's total behind them)
//   k_rpc_expand   one thread per decision of [lo, hi): its RPC by binary search, its request into the staged queue
//   ...            the staged solve, 8-byte grants left in HBM
//   k_rpc_grants   per RPC: its grants (a prefix of its decisions: a binary search), the status mapping
//   (k_scan_u32    exclusive scan of the grant counts: first_grant)
//   k_rpc_report   per RPC: first_grant; per granted decision: the grant to grants_out[ordinal]
//
// Why the report is a scatter by ordinal: all decisions of an RPC share class and requestor, failed decisions change no
// state, and within a batch running_tasks only grows, so a class that failed once keeps failing.  A granted decision
// therefore never follows a failed one of its own RPC: every grant of the window is reported, in FIFO order, and the k-th
// reported grant has ordinal k.  A grant outside its RPC's leading run (or with another ordinal) breaks that argument:
// k_rpc_report marks the RPC in its `reserved` word and the host aborts.
#pragma once
#include "common.cuh"
#include "radix.cuh"  // k_scan_u32

namespace yd {

// scheduler_service_impl.cc:221-226: over the limits nothing is attempted (INVALID_ARGUMENT)
__device__ __forceinline__ bool rpc_valid(const yd_rpc_wait& r) {
  return r.milliseconds_to_wait <= 10000u && r.next_keep_alive_ns <= 30000000000ll;
}
// ClampReqs: after `bound` grants in a batch the next decision fails, and nothing after an RPC's first failure is reported
__device__ __forceinline__ uint32_t rpc_clamp(uint32_t asked, unsigned long long bound) {
  return (uint32_t)min((unsigned long long)asked, bound + 1);
}

// The RPC decision q belongs to: the last i with off[i] <= q (off[0] = 0 <= q < off[n]).
__device__ __forceinline__ uint32_t rpc_of(const uint32_t* __restrict__ off, uint32_t n, uint32_t q) {
  uint32_t a = 0, b = n;
  while (b - a > 1) {
    const uint32_t m = (a + b) >> 1;
    if (off[m] <= q) a = m; else b = m;
  }
  return a;
}

__device__ __forceinline__ bool granted8(uint2 g) { return (g.y >> 30) == YD_STATUS_GRANTED; }

// off[0 .. n] = decisions per RPC, 0 at the end (the scan's end cell).  The host checked that the window's total fits.
__global__ void __launch_bounds__(256) k_rpc_count(const yd_rpc_wait* __restrict__ rpcs, uint32_t n,
                                                   unsigned long long bound, uint32_t* __restrict__ off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) off[n] = 0;
  if (i >= n) return;
  const yd_rpc_wait r = rpcs[i];
  off[i] = rpc_valid(r) ? rpc_clamp(r.immediate_reqs, bound) + rpc_clamp(r.prefetch_reqs, bound) : 0u;
}

// Decisions [lo, hi) of the window as requests, at out[0 .. hi - lo): each RPC asks for its immediate requests, then its
// prefetch requests.
__global__ void __launch_bounds__(256) k_rpc_expand(const yd_rpc_wait* __restrict__ rpcs, uint32_t n,
                                                    unsigned long long bound, const uint32_t* __restrict__ off, uint32_t lo,
                                                    uint32_t hi, yd_task_req* __restrict__ out) {
  const uint32_t q = lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= hi) return;
  const uint32_t i = rpc_of(off, n, q);
  const yd_rpc_wait r = rpcs[i];
  const bool prefetch = q - off[i] >= rpc_clamp(r.immediate_reqs, bound);
  out[q - lo] = yd_task_req{r.env_id, r.min_version, r.requestor_ip, prefetch ? YD_REQ_FLAG_PREFETCH : 0u,
                            r.next_keep_alive_ns};
}

// Per RPC, over the window's 8-byte grants g[0 .. off[n]): results[i] without first_grant, and its grant count in
// ng[i] (ng[n] = 0: the scan's end cell).  The grants of an RPC are a prefix of its decisions (above), so their count is
// where the first non-granted decision is.
__global__ void __launch_bounds__(256) k_rpc_grants(const yd_rpc_wait* __restrict__ rpcs, uint32_t n,
                                                    const uint32_t* __restrict__ off, const uint2* __restrict__ g,
                                                    uint32_t* __restrict__ ng, yd_rpc_wait_result* __restrict__ res) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) ng[n] = 0;
  if (i >= n) return;
  const yd_rpc_wait r = rpcs[i];
  const uint32_t b = off[i], e = off[i + 1];
  uint32_t a = b, z = e;
  while (a < z) {
    const uint32_t m = a + ((z - a) >> 1);
    if (granted8(g[m])) a = m + 1; else z = m;
  }
  const uint32_t k = a - b;
  uint32_t status = YD_RPC_OK;
  if (!rpc_valid(r)) {
    status = YD_RPC_INVALID_ARGUMENT;
  } else if (k == 0) {
    // :242-246: EnvironmentNotFound on an IMMEDIATE request fails the RPC with 1006; on a prefetch request it is just
    // "no result" (:260-262) and the RPC ends in 1001 (:266-270)
    const bool env_missing = e != b && (g[b].y >> 30) == YD_STATUS_ENVIRONMENT_NOT_FOUND && r.immediate_reqs != 0;
    status = env_missing ? YD_RPC_ENVIRONMENT_NOT_AVAILABLE : YD_RPC_NO_QUOTA_AVAILABLE;
  }
  res[i] = yd_rpc_wait_result{status, k, 0u, 0u};
  ng[i] = k;
}

// `first` = the scanned grant counts.  Thread t: first_grant of RPC t (t < n), and decision t's grant, if any, to
// out[its ordinal] (t < total).  A grant outside its RPC's leading run, or whose ordinal is not its place in the report,
// sets the RPC's `reserved` word instead.
__global__ void __launch_bounds__(256) k_rpc_report(uint32_t n, uint32_t total, const uint32_t* __restrict__ off,
                                                    const uint2* __restrict__ g, const uint32_t* __restrict__ first,
                                                    yd_rpc_wait_result* __restrict__ res, uint2* __restrict__ out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) res[t].first_grant = first[t];
  if (t >= total) return;
  const uint2 v = g[t];
  if (!granted8(v)) return;
  const uint32_t i = rpc_of(off, n, t);
  const uint32_t j = t - off[i], k = first[i] + j;
  if (j >= first[i + 1] - first[i] || (v.y & 0x3fffffffu) != k) {
    res[i].reserved = 1;
    return;
  }
  out[k] = v;
}

}  // namespace yd
