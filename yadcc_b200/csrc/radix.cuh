// radix.cuh -- stable LSD radix sort of (slot code, payload) pairs.
//
// Input order is (registry position, running_tasks) -- the order the slot table is
// generated in -- so a STABLE sort by code alone yields the reference's full pick
// order (tier, utilisation, registry position): ties on the code are broken by
// position exactly like `first minimum wins` (task_dispatcher.cc:444).
//
// One kernel up front counts the digits of ALL passes at once (the multiset of keys, hence
// every digit histogram, is the same before and after each permutation); then one kernel
// per pass: a block takes the next tile (ticket counter), counts its digits, publishes them,
// waits for the LOWER tiles' counts only (they are already running, so this cannot deadlock)
// and scatters.  base(digit, tile) = sum of all smaller digits (global histogram) + counts of
// that digit in lower tiles.  Stability inside a tile:
// warp w owns a contiguous chunk of the tile and walks it 32 elements at a time;
// __match_any_sync ranks equal digits inside a group, per-warp digit counters in
// shared memory carry the rank across groups, and a prefix over the warps' counts
// orders the warps.  Algorithmic bytes: keys read once by the histogram kernel; per pass
// keys read twice (count, scatter; the second read hits L1/L2) + payload once, both written once.
#pragma once
#include "common.cuh"

namespace yd {

constexpr int kRsBits = 7;
constexpr int kRsBins = 1 << kRsBits;
constexpr int kRsThreads = 256;
constexpr int kRsWarps = kRsThreads / 32;
constexpr int kRsItemsPerWarp = 128;                    // 4 groups of 32
constexpr int kRsTile = kRsWarps * kRsItemsPerWarp;     // 1024 elements per block (measured: 2048 is 5 % slower at 130 k keys)

template <typename KeyT>
__device__ __forceinline__ uint32_t rs_digit(KeyT k, int shift) {
  return (uint32_t)(k >> shift) & (kRsBins - 1);
}

constexpr int kScanItems8 = 8;

// Exclusive scan (in place) of a (rows x per_row) count matrix laid out row-major, + the grand total in the cell
// behind it -- the (class, tile) count tables of classes.cuh / parallel.cuh.  One block per row: the row is scanned
// on its own, its total published (a 64-bit word per row in `pub`, gridDim.x + 1 words zeroed by the caller: bit 63 = ready), the totals of
// the rows before it summed, and the base added in a second sweep.  rows = min(*n_rows_dyn, gridDim.x) blocks take
// part; they are co-resident (<= 256 blocks), so waiting for lower rows cannot dead-lock.
__global__ void __launch_bounds__(1024) k_scan_rows(uint32_t* __restrict__ data, const uint32_t* __restrict__ n_rows_dyn,
                                                    uint32_t per_row, unsigned long long* __restrict__ pub) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s, base_s, row_s;
  const uint32_t rows = min(*n_rows_dyn, gridDim.x);
  // rows are handed out by ticket (pub[gridDim.x]): whoever waits for a lower row knows that row is running
  if (threadIdx.x == 0) row_s = (uint32_t)atomicAdd(&pub[gridDim.x], 1ull);
  __syncthreads();
  const uint32_t row = row_s;
  if (row >= rows) return;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t* d = data + size_t(row) * per_row;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t b0 = 0; b0 < per_row; b0 += 1024 * kScanItems8) {
    const uint32_t i0 = b0 + tid * kScanItems8;
    uint32_t v[kScanItems8];
#pragma unroll
    for (int k = 0; k < kScanItems8; ++k) v[k] = (i0 + k < per_row) ? d[i0 + k] : 0;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < kScanItems8; ++k) sum += v[k];
    uint32_t x = sum;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, s);
      if (lane >= s) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = warp_sums[lane];
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, w, s);
        if (lane >= s) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const uint32_t carry = carry_s;
    uint32_t run = carry + (warp ? warp_sums[warp - 1] : 0) + x - sum;
#pragma unroll
    for (int k = 0; k < kScanItems8; ++k) {
      if (i0 + k < per_row) d[i0 + k] = run;
      run += v[k];
    }
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_sums[31];
    __syncthreads();
  }
  volatile unsigned long long* vp = pub;
  if (tid == 0) { __threadfence(); vp[row] = (1ull << 63) | carry_s; }
  if (warp == 0) {  // totals of the rows before mine
    uint32_t base = 0;
    for (uint32_t r0 = 0; r0 < row; r0 += 32) {
      const uint32_t r = r0 + lane;
      unsigned long long w = 1ull << 63;
      if (r < row) { do { w = vp[r]; } while (!(w >> 63)); }
      base += __reduce_add_sync(0xffffffffu, r < row ? (uint32_t)w : 0u);
    }
    if (lane == 0) base_s = base;
  }
  __syncthreads();
  const uint32_t base = base_s;
  if (base) {
    for (uint32_t i = tid; i < per_row; i += 1024) d[i] += base;
  }
  if (row == rows - 1 && tid == 0) data[size_t(rows) * per_row] = base + carry_s;  // the end cell
}

// Generic one-block exclusive scan (in place).  Each thread owns 8 consecutive
// values (two 16-byte loads), so 8192 values need one block-wide round.  The length
// is n_static, or min(*n_dyn, dyn_cap) * per_dyn + 1 when n_dyn != nullptr (sizes that only
// the device knows, e.g. number of classes x tiles; dyn_cap = what the buffer was sized for).
constexpr int kScanItems = 8;
__global__ void __launch_bounds__(1024) k_scan_u32(uint32_t* __restrict__ data, uint32_t n_static,
                                                   const uint32_t* __restrict__ n_dyn, uint32_t per_dyn,
                                                   uint32_t* __restrict__ total_out, uint32_t dyn_cap) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = n_dyn ? min(*n_dyn, dyn_cap) * per_dyn + 1 : n_static;  // never past what the host sized
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n; base += 1024 * kScanItems) {
    const uint32_t i0 = base + tid * kScanItems;
    uint32_t v[kScanItems];
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) v[k] = (i0 + k < n) ? data[i0 + k] : 0;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) sum += v[k];
    uint32_t x = sum;
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
    const uint32_t carry = carry_s;
    uint32_t run = carry + (warp ? warp_sums[warp - 1] : 0) + x - sum;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      if (i0 + k < n) data[i0 + k] = run;
      run += v[k];
    }
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_sums[31];
    __syncthreads();
  }
  if (tid == 0 && total_out) *total_out = carry_s;
}

// ---- onesweep-style passes -----------------------------------------------------------------

constexpr int kRsMaxPasses = 9;  // 63 key bits / 7

// Scratch of one pass inside the zero-initialised region (32-bit words).
struct RsPassScratch {
  uint32_t* tile_hist;  // [nb][kRsBins] digit counts per tile, stored as count + 1 (0 = not published yet)
  uint32_t* ticket;     // [1]  next tile to hand out
  uint32_t* ghist;      // [kRsBins] digit counts over all keys (k_rs_ghist)
};
__host__ __device__ inline size_t rs_pass_words(uint32_t nb) {
  return ((size_t(kRsBins) * nb + kRsBins + 1) + 3) & ~size_t(3);
}
__host__ __device__ inline RsPassScratch rs_pass_scratch(uint32_t* base, uint32_t nb) {
  RsPassScratch r;
  r.tile_hist = base;                      // 16-byte aligned: region sizes are multiples of 4 words
  r.ghist = base + size_t(kRsBins) * nb;
  r.ticket = r.ghist + kRsBins;
  return r;
}

// Digit histograms of every pass in one read of the keys.
template <typename KeyT>
__global__ void __launch_bounds__(kRsThreads) k_rs_ghist(const KeyT* __restrict__ keys,
                                                         const unsigned long long* __restrict__ n_ptr, int first_bit,
                                                         int passes, uint32_t nb, uint32_t* __restrict__ zbase) {
  __shared__ uint32_t h[kRsMaxPasses][kRsBins];
  const uint32_t n = (uint32_t)*n_ptr;
  for (int i = threadIdx.x; i < passes * kRsBins; i += kRsThreads) (&h[0][0])[i] = 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * kRsTile;
  for (uint32_t i = threadIdx.x; i < kRsTile; i += kRsThreads) {
    const uint32_t g = base + i;
    if (g < n) {
      const KeyT k = keys[g];
      for (int p = 0; p < passes; ++p) atomicAdd(&h[p][rs_digit(k, first_bit + p * kRsBits)], 1u);
    }
  }
  __syncthreads();
  const size_t stride = rs_pass_words(nb);
  for (int i = threadIdx.x; i < passes * kRsBins; i += kRsThreads) {
    const uint32_t c = (&h[0][0])[i];
    if (c) atomicAdd(rs_pass_scratch(zbase + (i / kRsBins) * stride, nb).ghist + (i % kRsBins), c);
  }
}

// 16-byte load that always goes to L2 (the words are written by other SMs during this kernel).
__device__ __forceinline__ uint4 rs_ld_volatile_v4(const uint32_t* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

template <typename KeyT>
__global__ void __launch_bounds__(kRsThreads) k_rs_pass(const KeyT* __restrict__ keys_in,
                                                        const uint32_t* __restrict__ vals_in,
                                                        const unsigned long long* __restrict__ n_ptr, int shift,
                                                        uint32_t nb, RsPassScratch sc, KeyT* __restrict__ keys_out,
                                                        uint32_t* __restrict__ vals_out) {
  __shared__ uint32_t wcnt[kRsWarps][kRsBins];  // per-warp digit counts, then running offsets
  __shared__ uint32_t dig_base[kRsBins];        // global base of (digit, this tile)
  __shared__ uint32_t wsum[kRsThreads / 32];
  __shared__ uint32_t part[kRsWarps][kRsBins];  // look-back partial sums per warp
  __shared__ uint32_t s_tile;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = (uint32_t)*n_ptr;
  // A pass in which every key has the same digit is the identity permutation (the sort is
  // stable): just move the tile to the output buffer.  Typical for the low fraction bits when
  // capacities are powers of two.  All blocks see the same histogram, so all take this branch.
  if (n != 0 && sc.ghist[rs_digit(keys_in[0], shift)] == n) {
    const uint32_t base = blockIdx.x * kRsTile;
    for (uint32_t i = tid; i < kRsTile; i += kRsThreads) {
      const uint32_t idx = base + i;
      if (idx < n) {
        keys_out[idx] = keys_in[idx];
        vals_out[idx] = vals_in ? vals_in[idx] : idx;
      }
    }
    return;
  }
  if (tid == 0) s_tile = atomicAdd(sc.ticket, 1u);  // tiles are handed out in start order
  for (int i = tid; i < kRsWarps * kRsBins; i += kRsThreads) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t wbase = tile * kRsTile + warp * kRsItemsPerWarp;
  // pass 1: count digits of my chunk
  for (int g = 0; g < kRsItemsPerWarp; g += 32) {
    uint32_t idx = wbase + g + lane;
    if (idx < n) atomicAdd(&wcnt[warp][rs_digit(keys_in[idx], shift)], 1u);
  }
  __syncthreads();
  // Publish this tile's digit counts as count + 1: every word validates itself (0 = not there
  // yet), so no flag and no fence are needed.
  if (tid < kRsBins) {
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < kRsWarps; ++w) c += wcnt[w][tid];
    __stcg(sc.tile_hist + size_t(tile) * kRsBins + tid, c + 1);
  }
  // Look back: counts of every digit in the LOWER tiles (all of them are running: they drew their
  // ticket before us).  Warp w takes tiles w, w + 8, ...; a lane owns four digits (one 16-byte
  // load per tile); four tiles are in flight per round.
  {
    uint4 acc = make_uint4(0, 0, 0, 0);
    static_assert(kRsBins == 128, "a lane owns kRsBins / 32 = 4 digits");
    for (uint32_t b0 = warp; b0 < tile; b0 += kRsWarps * 4) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t b = b0 + j * kRsWarps;
        v[j] = b < tile ? rs_ld_volatile_v4(sc.tile_hist + size_t(b) * kRsBins + lane * 4) : make_uint4(1, 1, 1, 1);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t b = b0 + j * kRsWarps;
        while (v[j].x == 0 || v[j].y == 0 || v[j].z == 0 || v[j].w == 0) {
          v[j] = rs_ld_volatile_v4(sc.tile_hist + size_t(b) * kRsBins + lane * 4);
        }
        acc.x += v[j].x - 1; acc.y += v[j].y - 1; acc.z += v[j].z - 1; acc.w += v[j].w - 1;
      }
    }
    part[warp][lane * 4 + 0] = acc.x; part[warp][lane * 4 + 1] = acc.y;
    part[warp][lane * 4 + 2] = acc.z; part[warp][lane * 4 + 3] = acc.w;
  }
  __syncthreads();
  {
    uint32_t total = 0, before = 0;
    if (tid < kRsBins) {
      total = sc.ghist[tid];
#pragma unroll
      for (int w = 0; w < kRsWarps; ++w) before += part[w][tid];
    }
    // exclusive scan of `total` over the digits (kRsBins <= kRsThreads)
    uint32_t x = total;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    uint32_t woff = 0;
    for (uint32_t w = 0; w < warp; ++w) woff += wsum[w];
    if (tid < kRsBins) dig_base[tid] = woff + x - total + before;
    __syncthreads();
  }
  // per digit: exclusive prefix over warps, offset by this tile's global base
  for (int d = tid; d < kRsBins; d += kRsThreads) {
    uint32_t run = dig_base[d];
#pragma unroll
    for (int w = 0; w < kRsWarps; ++w) {
      uint32_t c = wcnt[w][d];
      wcnt[w][d] = run;
      run += c;
    }
  }
  __syncthreads();
  // pass 2: stable ranks inside my chunk, group by group
  for (int g = 0; g < kRsItemsPerWarp; g += 32) {
    uint32_t idx = wbase + g + lane;
    bool valid = idx < n;
    KeyT k = valid ? keys_in[idx] : (KeyT)0;
    uint32_t d = valid ? rs_digit(k, shift) : (uint32_t)kRsBins;  // invalid lanes form their own group
    uint32_t peers = __match_any_sync(0xffffffffu, d);
    uint32_t rank = __popc(peers & ((1u << lane) - 1));
    uint32_t dst = 0;
    if (valid) dst = wcnt[warp][d] + rank;
    __syncwarp();
    if (valid && rank == 0) wcnt[warp][d] += __popc(peers);  // leader advances the running offset
    __syncwarp();
    if (valid) {
      keys_out[dst] = k;
      vals_out[dst] = vals_in ? vals_in[idx] : idx;  // first pass: payload = original slot index
    }
  }
}

// The whole sort on `st`: stable by bits [first_bit, first_bit + 7 * passes) of the keys, passes = (last_bit - first_bit)
// / 7 + 1, payloads starting as the keys' indices.  n = *n_ptr (known on the device only), nb >= ceil(n / kRsTile) tiles.
// The digit histograms of all passes in one read, then one kernel per pass, ping-ponging between buffers 0 and 1 of
// keys_out / vals_out so that the LAST pass writes buffer 0 (captured graphs keep its address); keys_in is only read.
// zbase: rs_pass_words(nb) words per pass, zeroed by the caller.  Returns the number of kernels launched.
template <typename KeyT>
inline uint32_t rs_sort(const KeyT* keys_in, const unsigned long long* n_ptr, uint32_t nb, int first_bit, int last_bit,
                        uint32_t* zbase, KeyT* const keys_out[2], uint32_t* const vals_out[2], cudaStream_t st) {
  const size_t stride = rs_pass_words(nb);
  const int passes = (last_bit - first_bit) / kRsBits + 1;
  const KeyT* kin = keys_in;
  const uint32_t* vin = nullptr;
  int cur = (passes - 1) & 1;
  k_rs_ghist<KeyT><<<nb, kRsThreads, 0, st>>>(kin, n_ptr, first_bit, passes, nb, zbase);
  for (int pass = 0; pass < passes; ++pass) {
    k_rs_pass<KeyT><<<nb, kRsThreads, 0, st>>>(kin, vin, n_ptr, first_bit + pass * kRsBits, nb,
                                               rs_pass_scratch(zbase + pass * stride, nb), keys_out[cur], vals_out[cur]);
    kin = keys_out[cur];
    vin = vals_out[cur];
    cur ^= 1;
  }
  return 1 + passes;
}

}  // namespace yd
