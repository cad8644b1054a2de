// First-party stable LSD radix sort of (int64 key, uint32 item) pairs and run-head compaction,
// the two device-wide primitives of the deduplicated sparse update (the reference takes them
// from CUB: embedding_lookup_kernels.cu:645-661).
//
// Keys are sorted as uint32 when every row key fits 32 bits (the common case: < 4 G rows per
// rank), which cuts the traffic per pass from 32 to 20 bytes per pair.
// Sort: 8-bit digits, three kernels per pass:
//   1. digit_hist_kernel    per-tile digit histogram -> hist[digit][tile]
//   2. digit_scan_kernel    one block per digit: exclusive scan of its row over the tiles
//   3. digit_scatter_kernel stable in-tile ranking with warp match_any multi-split, then
//                           scatter to digit_base + tile_offset + in-tile rank
// A tile is 4096 consecutive pairs ordered (warp, round, lane); every level preserves that order,
// so equal keys keep their input order (the update kernels rely on deterministic item order).
// Only bits [0, end_bit) are sorted: callers pass bit_length(total_rows).
//
// Heads: flag[i] = (i == 0 || key[i] != key[i-1]); count per tile, scan the tile counts in one
// block, then compact the positions of the heads in order -> seg_start, n_unique.
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "de_b200.h"

namespace de {
namespace {

constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kRounds = 16;  // pairs per thread
constexpr int kSortTile = kSortThreads * kRounds;
constexpr int kBins = 256;
constexpr int kScanThreads = 1024;

__device__ __forceinline__ uint32_t lanemask_lt() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// exclusive scan of one value per thread over the block; returns the exclusive prefix and the
// block total through `total` (same on every thread).  `warp_sums` holds blockDim.x / 32 words.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums,
                                                         uint32_t& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t s = lane < n_warps ? warp_sums[lane] : 0u;
    uint32_t si = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, si, d);
      if (lane >= d) si += t;
    }
    if (lane < n_warps) warp_sums[lane] = si - s;  // exclusive warp base
    if (lane == 31) warp_sums[32] = si;            // block total
  }
  __syncthreads();
  uint32_t base = warp_sums[warp];
  total = warp_sums[32];
  __syncthreads();  // warp_sums may be reused by the caller's next scan
  return base + incl - v;
}

template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads)
    digit_hist_kernel(const KeyT* __restrict__ keys, int64_t n, int shift, int64_t n_tiles,
                      uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[kBins];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile;
#pragma unroll 4
  for (int r = 0; r < kRounds; ++r) {
    int64_t i = base + r * kSortThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & (kBins - 1)], 1u);
  }
  __syncthreads();
  hist[static_cast<int64_t>(threadIdx.x) * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// block d: hist[d][0..n_tiles) -> exclusive prefix in place, total[d] = row sum
__global__ void __launch_bounds__(kScanThreads)
    digit_scan_kernel(uint32_t* __restrict__ hist, int64_t n_tiles, uint32_t* __restrict__ total) {
  __shared__ uint32_t warp_sums[33];
  uint32_t* row = hist + static_cast<int64_t>(blockIdx.x) * n_tiles;
  uint32_t carry = 0;
  for (int64_t c = 0; c < n_tiles; c += kScanThreads) {
    int64_t i = c + threadIdx.x;
    uint32_t v = i < n_tiles ? row[i] : 0u;
    uint32_t chunk;
    uint32_t ex = block_exclusive_scan(v, warp_sums, chunk);
    if (i < n_tiles) row[i] = carry + ex;
    carry += chunk;
  }
  if (threadIdx.x == 0) total[blockIdx.x] = carry;
}

// KeyIn / KeyOut: int64 keys, or uint32 keys when every row key fits 32 bits (8 instead of 12
// bytes per pair and pass); the last pass of a 32-bit sort widens to the int64 keys the update
// kernels consume (KeyOut = int64_t).  kItems = false: keys only (items_in / items_out unused).
template <typename KeyIn, typename KeyOut, bool kItems = true>
__global__ void __launch_bounds__(kSortThreads)
    digit_scatter_kernel(const KeyIn* __restrict__ keys_in, const uint32_t* __restrict__ items_in,
                         KeyOut* __restrict__ keys_out, uint32_t* __restrict__ items_out,
                         int64_t n, int shift, int64_t n_tiles, const uint32_t* __restrict__ hist,
                         const uint32_t* __restrict__ total) {
  __shared__ uint32_t warp_cnt[kSortWarps][kBins];
  __shared__ uint32_t warp_sums[33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // global start of every digit's run for this tile
  uint32_t tot;
  uint32_t digit_base = block_exclusive_scan(total[threadIdx.x], warp_sums, tot) +
                        hist[static_cast<int64_t>(threadIdx.x) * n_tiles + blockIdx.x];
#pragma unroll
  for (int w = 0; w < kSortWarps; ++w) warp_cnt[w][threadIdx.x] = 0;
  __syncthreads();

  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + warp * (kRounds * 32) + lane;
  KeyIn key[kRounds];
  uint32_t item[kRounds];
  uint32_t rank[kRounds];
  const uint32_t lt = lanemask_lt();
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    int64_t i = base + r * 32;
    bool valid = i < n;
    key[r] = valid ? keys_in[i] : 0;
    item[r] = kItems && valid ? items_in[i] : 0u;
  }
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    bool valid = base + r * 32 < n;
    uint32_t d = valid ? static_cast<uint32_t>((key[r] >> shift) & (kBins - 1)) : kBins;
    uint32_t peers = __match_any_sync(0xffffffffu, d);
    int leader = __ffs(peers) - 1;
    uint32_t old = 0;
    if (lane == leader && valid) {
      old = warp_cnt[warp][d];
      warp_cnt[warp][d] = old + __popc(peers);
    }
    old = __shfl_sync(0xffffffffu, old, leader);
    rank[r] = old + __popc(peers & lt);
    __syncwarp();
  }
  __syncthreads();
  {
    // digit threadIdx.x: turn per-warp counts into per-warp global bases
    uint32_t run = digit_base;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) {
      uint32_t c = warp_cnt[w][threadIdx.x];
      warp_cnt[w][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    if (base + r * 32 < n) {
      uint32_t d = static_cast<uint32_t>((key[r] >> shift) & (kBins - 1));
      uint32_t pos = warp_cnt[warp][d] + rank[r];
      keys_out[pos] = static_cast<KeyOut>(key[r]);
      if (kItems) items_out[pos] = item[r];
    }
  }
}

// ---- heads ---------------------------------------------------------------------------------
// tile order is (warp, round, lane) like the sort; ballots are warp-uniform so the in-warp rank
// of a head is popc(ballot & lanemask_lt) + heads in the warp's earlier rounds.
__device__ __forceinline__ uint32_t head_ballot(const int64_t* __restrict__ keys, int64_t i,
                                                int64_t n) {
  bool head = false;
  if (i < n) head = (i == 0) || (keys[i] != keys[i - 1]);
  return __ballot_sync(0xffffffffu, head);
}

__global__ void __launch_bounds__(kSortThreads)
    head_count_kernel(const int64_t* __restrict__ keys, int64_t n, uint32_t* __restrict__ tile_count) {
  __shared__ uint32_t warp_tot[kSortWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + warp * (kRounds * 32) + lane;
  uint32_t c = 0;
#pragma unroll 4
  for (int r = 0; r < kRounds; ++r) c += __popc(head_ballot(keys, base + r * 32, n));
  if (lane == 0) warp_tot[warp] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) s += warp_tot[w];
    tile_count[blockIdx.x] = s;
  }
}

// single block: tile_count -> exclusive prefix in place; n_unique; seg_start[n_unique] = n
__global__ void __launch_bounds__(kScanThreads)
    head_scan_kernel(uint32_t* __restrict__ tile_count, int64_t n_tiles, int64_t n,
                     int64_t* __restrict__ seg_start, int64_t* __restrict__ n_unique) {
  __shared__ uint32_t warp_sums[33];
  uint32_t carry = 0;
  for (int64_t c = 0; c < n_tiles; c += kScanThreads) {
    int64_t i = c + threadIdx.x;
    uint32_t v = i < n_tiles ? tile_count[i] : 0u;
    uint32_t chunk;
    uint32_t ex = block_exclusive_scan(v, warp_sums, chunk);
    if (i < n_tiles) tile_count[i] = carry + ex;
    carry += chunk;
  }
  if (threadIdx.x == 0) {
    *n_unique = carry;
    seg_start[carry] = n;
  }
}

__global__ void __launch_bounds__(kSortThreads)
    head_compact_kernel(const int64_t* __restrict__ keys, int64_t n,
                        const uint32_t* __restrict__ tile_off, int64_t* __restrict__ seg_start) {
  __shared__ uint32_t warp_tot[kSortWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + warp * (kRounds * 32) + lane;
  uint32_t ballots[kRounds];
  uint32_t c = 0;
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    ballots[r] = head_ballot(keys, base + r * 32, n);
    c += __popc(ballots[r]);
  }
  if (lane == 0) warp_tot[warp] = c;
  __syncthreads();
  uint32_t run = tile_off[blockIdx.x];
  for (int w = 0; w < warp; ++w) run += warp_tot[w];
  const uint32_t lt = lanemask_lt();
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    if ((ballots[r] >> lane) & 1u) seg_start[run + __popc(ballots[r] & lt)] = base + r * 32;
    run += __popc(ballots[r]);
  }
}

inline int64_t tiles_of(int64_t n) { return (n + kSortTile - 1) / kSortTile; }
inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

}  // namespace

size_t radix_sort_temp_bytes(int64_t n) {
  return align256(static_cast<size_t>(tiles_of(n)) * kBins * sizeof(uint32_t)) +
         align256(kBins * sizeof(uint32_t));
}

// Sorts bits [0, end_bit) with ping-pong between (keys_a, items_a) and (keys_b, items_b); both
// pairs are clobbered.  Returns 0 when the sorted pairs end in a, 1 when they end in b.
int radix_sort_pairs(void* temp, int64_t* keys_a, uint32_t* items_a, int64_t* keys_b,
                     uint32_t* items_b, int64_t n, int end_bit, cudaStream_t stream) {
  if (n <= 0) return 0;
  const int64_t n_tiles = tiles_of(n);
  uint32_t* hist = static_cast<uint32_t*>(temp);
  uint32_t* total = reinterpret_cast<uint32_t*>(
      static_cast<char*>(temp) + align256(static_cast<size_t>(n_tiles) * kBins * sizeof(uint32_t)));
  int64_t* kin = keys_a;
  uint32_t* iin = items_a;
  int64_t* kout = keys_b;
  uint32_t* iout = items_b;
  int where = 0;
  if (end_bit < 1) end_bit = 1;
  for (int shift = 0; shift < end_bit; shift += 8) {
    digit_hist_kernel<int64_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0, stream>>>(
        kin, n, shift, n_tiles, hist);
    digit_scan_kernel<<<kBins, kScanThreads, 0, stream>>>(hist, n_tiles, total);
    digit_scatter_kernel<int64_t, int64_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0,
                                             stream>>>(kin, iin, kout, iout, n, shift, n_tiles,
                                                       hist, total);
    int64_t* tk = kin;
    kin = kout;
    kout = tk;
    uint32_t* ti = iin;
    iin = iout;
    iout = ti;
    where ^= 1;
  }
  return where;
}

// 32-bit keys (every key < 2^32): same passes on (uint32 key, uint32 item) pairs, the last pass
// writes the keys widened to int64 into keys_out64.  Returns which items buffer holds the sorted
// items (0: items_a, 1: items_b).  keys_a / keys_b are clobbered.
int radix_sort_pairs32(void* temp, uint32_t* keys_a, uint32_t* items_a, uint32_t* keys_b,
                       uint32_t* items_b, int64_t* keys_out64, int64_t n, int end_bit,
                       cudaStream_t stream) {
  if (n <= 0) return 0;
  const int64_t n_tiles = tiles_of(n);
  uint32_t* hist = static_cast<uint32_t*>(temp);
  uint32_t* total = reinterpret_cast<uint32_t*>(
      static_cast<char*>(temp) + align256(static_cast<size_t>(n_tiles) * kBins * sizeof(uint32_t)));
  uint32_t *kin = keys_a, *iin = items_a, *kout = keys_b, *iout = items_b;
  int where = 0;
  if (end_bit < 1) end_bit = 1;
  if (end_bit > 32) end_bit = 32;
  for (int shift = 0; shift < end_bit; shift += 8) {
    const bool last = shift + 8 >= end_bit;
    digit_hist_kernel<uint32_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0, stream>>>(
        kin, n, shift, n_tiles, hist);
    digit_scan_kernel<<<kBins, kScanThreads, 0, stream>>>(hist, n_tiles, total);
    if (last)
      digit_scatter_kernel<uint32_t, int64_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0,
                                                stream>>>(kin, iin, keys_out64, iout, n, shift,
                                                          n_tiles, hist, total);
    else
      digit_scatter_kernel<uint32_t, uint32_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0,
                                                 stream>>>(kin, iin, kout, iout, n, shift, n_tiles,
                                                           hist, total);
    uint32_t* tk = kin;
    kin = kout;
    kout = tk;
    uint32_t* ti = iin;
    iin = iout;
    iout = ti;
    where ^= 1;
  }
  return where;
}

// Keys only (every key < 2^32): the passes of radix_sort_pairs32 without items, ping-pong
// between keys_a and keys_b (both clobbered).  Returns 0 when the sorted keys end in keys_a, 1
// when they end in keys_b.
int radix_sort_keys32(void* temp, uint32_t* keys_a, uint32_t* keys_b, int64_t n, int end_bit,
                      cudaStream_t stream) {
  if (n <= 0) return 0;
  const int64_t n_tiles = tiles_of(n);
  uint32_t* hist = static_cast<uint32_t*>(temp);
  uint32_t* total = reinterpret_cast<uint32_t*>(
      static_cast<char*>(temp) + align256(static_cast<size_t>(n_tiles) * kBins * sizeof(uint32_t)));
  uint32_t *kin = keys_a, *kout = keys_b;
  int where = 0;
  if (end_bit < 1) end_bit = 1;
  if (end_bit > 32) end_bit = 32;
  for (int shift = 0; shift < end_bit; shift += 8) {
    digit_hist_kernel<uint32_t><<<static_cast<unsigned>(n_tiles), kSortThreads, 0, stream>>>(
        kin, n, shift, n_tiles, hist);
    digit_scan_kernel<<<kBins, kScanThreads, 0, stream>>>(hist, n_tiles, total);
    digit_scatter_kernel<uint32_t, uint32_t, false><<<static_cast<unsigned>(n_tiles),
                                                      kSortThreads, 0, stream>>>(
        kin, nullptr, kout, nullptr, n, shift, n_tiles, hist, total);
    uint32_t* tk = kin;
    kin = kout;
    kout = tk;
    where ^= 1;
  }
  return where;
}

size_t head_segments_temp_bytes(int64_t n) {
  return align256(static_cast<size_t>(tiles_of(n)) * sizeof(uint32_t));
}

void head_segments(void* temp, const int64_t* sorted_keys, int64_t n, int64_t* seg_start,
                   int64_t* n_unique, cudaStream_t stream) {
  if (n <= 0) {
    cudaMemsetAsync(n_unique, 0, sizeof(int64_t), stream);
    return;
  }
  const int64_t n_tiles = tiles_of(n);
  uint32_t* tile_count = static_cast<uint32_t*>(temp);
  head_count_kernel<<<static_cast<unsigned>(n_tiles), kSortThreads, 0, stream>>>(sorted_keys, n,
                                                                                 tile_count);
  head_scan_kernel<<<1, kScanThreads, 0, stream>>>(tile_count, n_tiles, n, seg_start, n_unique);
  head_compact_kernel<<<static_cast<unsigned>(n_tiles), kSortThreads, 0, stream>>>(
      sorted_keys, n, tile_count, seg_start);
}

}  // namespace de
