// HBM row cache of host-offloaded (pinned, zero-copy) fp32 tables, sm_90a.
//
// A cached table keeps `n_sets` sets of 32 ways plus a spill region of `n_spill` slots in HBM:
// weight rows and their optimizer-state rows, one int64 tag (host row or -1) per slot, one
// last-use tick per way and one dirty word per slot.  Each step the cache pass
//   1. writes the dirty rows of the previous step's spill region back to the host and empties it;
//   2. finds the unique rows the step touches (build_keys + first-party radix sort + heads);
//   3. probe:  one warp per unique row ballots over the 32 tags of the row's set; a hit refreshes
//              the way's tick (and sets the dirty bit in a training pass);
//   4. sorts the misses by set (stable: a set's misses stay in ascending row order) and finds the
//      per-set runs;
//   5. assign: one warp per set run gives the misses the set's least recently used ways (ties by
//              way index), never a way used in this tick; the rest go to spill slot
//              n_sets * 32 + u (u = the row's unique index), so every row of the step has a slot;
//   6. fill:   one warp per miss writes the evicted dirty row back, then copies the new row (and
//              its state) from the host, 16 bytes per lane access, through the UVA mapping;
//   7. remap:  every id of the cached inputs becomes its slot id (-1 for out-of-shard ids) in a
//              buffer laid out like the owner's id buffer.
// The policy is defined in parallel/offload_cache.py; tests compare the two exactly.
// Grids are fixed by the static bound on unique rows (the unique count stays on the device), so
// the pass captures in a CUDA graph.
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "de_b200.h"

namespace de {
namespace {

constexpr int kCacheThreads = 256;
constexpr int kCacheWarps = kCacheThreads / 32;

// the set of a row: murmur3 fmix64-style mixing, mod the number of sets (cache_set in Python)
__device__ __forceinline__ int64_t cache_set(int64_t row, int64_t n_sets) {
  uint64_t x = static_cast<uint64_t>(row);
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  return static_cast<int64_t>(x % static_cast<uint64_t>(n_sets));
}

// one warp copies `width` fp32 words; vec: width % 4 == 0 and both rows 16-byte aligned
__device__ __forceinline__ void warp_copy_row(float* __restrict__ dst, const float* __restrict__ src,
                                              int width, bool vec, int lane) {
  if (vec) {
    const float4* s = reinterpret_cast<const float4*>(src);
    float4* d = reinterpret_cast<float4*>(dst);
    for (int c = lane; c < width / 4; c += 32) d[c] = s[c];
  } else {
    for (int c = lane; c < width; c += 32) dst[c] = src[c];
  }
}

// the weight row and every state row of cache slot `slot` <-> host row `row`
__device__ __forceinline__ void move_row(const CacheTable& T, int64_t slot, int64_t row,
                                         bool to_host, int lane) {
  const int64_t w = T.width;
  const bool vec = (w & 3) == 0;
  if (to_host) {
    warp_copy_row(T.host_weight + row * w, T.weight + slot * w, T.width, vec, lane);
  } else {
    warp_copy_row(T.weight + slot * w, T.host_weight + row * w, T.width, vec, lane);
  }
  const int sw[2] = {T.state0_width, T.state1_width};
  float* const cs[2] = {T.state0, T.state1};
  float* const hs[2] = {T.host_state0, T.host_state1};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (sw[k] <= 0) continue;
    const int64_t s = sw[k];
    const bool v = (s & 3) == 0;
    if (to_host) warp_copy_row(hs[k] + row * s, cs[k] + slot * s, sw[k], v, lane);
    else warp_copy_row(cs[k] + slot * s, hs[k] + row * s, sw[k], v, lane);
  }
}

// 1. previous step's spill region -> host (dirty rows), then empty it
__global__ void __launch_bounds__(kCacheThreads)
    cache_spill_writeback_kernel(const __grid_constant__ CacheTable T) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kCacheWarps;
  const int64_t base = T.n_sets * 32;
  for (int64_t s = warp; s < T.n_spill; s += n_warps) {
    const int64_t slot = base + s;
    const int64_t row = T.tags[slot];
    if (row < 0) continue;
    if (T.dirty[slot]) {
      move_row(T, slot, row, true, lane);
      if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[3]), 1ull);
    }
    __syncwarp();
    if (lane == 0) {
      T.tags[slot] = -1;
      T.dirty[slot] = 0;
    }
  }
}

// 3. probe.  uniq[u] = row of unique u (rows for u >= n_unique); miss_set[u] = set of a miss,
// n_sets otherwise (sorts behind every set); move[u] = -2 (no fill) until assign decides.
__global__ void __launch_bounds__(kCacheThreads)
    cache_probe_kernel(const __grid_constant__ CacheTable T, const int64_t* __restrict__ sorted_keys,
                       const int64_t* __restrict__ seg_start, const int64_t* __restrict__ n_unique,
                       int64_t cap, int train, int64_t* __restrict__ uniq,
                       uint32_t* __restrict__ miss_set, uint32_t* __restrict__ miss_item,
                       int64_t* __restrict__ slot_of, int64_t* __restrict__ move) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kCacheWarps;
  const int64_t nu = *n_unique;
  const int32_t now = *T.tick_word + 1;
  for (int64_t u = warp; u < cap; u += n_warps) {
    const int64_t key = u < nu ? sorted_keys[seg_start[u]] : T.rows;
    uint32_t set_out = static_cast<uint32_t>(T.n_sets);
    int64_t slot_out = -1;
    if (key < T.rows) {
      const int64_t set = cache_set(key, T.n_sets);
      const int64_t slot = set * 32 + lane;
      const uint32_t hit = __ballot_sync(0xffffffffu, T.tags[slot] == key);
      if (hit) {
        const int way = __ffs(hit) - 1;
        slot_out = set * 32 + way;
        if (lane == way) {
          T.ticks[slot_out] = now;
          if (train) T.dirty[slot_out] = 1;
          atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[0]), 1ull);
        }
      } else {
        set_out = static_cast<uint32_t>(set);
      }
    }
    if (lane == 0) {
      uniq[u] = key;
      miss_set[u] = set_out;
      miss_item[u] = static_cast<uint32_t>(u);
      slot_of[u] = slot_out;
      move[u] = -2;
    }
  }
}

// 5. assign.  set_sorted / u_sorted: misses sorted by set; seg / n_seg: the per-set runs.
__global__ void __launch_bounds__(kCacheThreads)
    cache_assign_kernel(const __grid_constant__ CacheTable T, const int64_t* __restrict__ set_sorted,
                        const uint32_t* __restrict__ u_sorted, const int64_t* __restrict__ seg,
                        const int64_t* __restrict__ n_seg, int64_t cap, int train,
                        const int64_t* __restrict__ uniq, int64_t* __restrict__ slot_of,
                        int64_t* __restrict__ move) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kCacheWarps;
  const int64_t ns = *n_seg;
  const int32_t now = *T.tick_word + 1;
  for (int64_t j = warp; j < ns && j < cap; j += n_warps) {
    const int64_t first = seg[j];
    const int64_t set = set_sorted[first];
    if (set >= T.n_sets) continue;  // the run of hits / invalid rows
    const int64_t count = seg[j + 1] - first;
    const int64_t slot = set * 32 + lane;
    const int32_t tick = T.ticks[slot];
    const bool avail = tick != now;
    const uint32_t avail_mask = __ballot_sync(0xffffffffu, avail);
    const int n_avail = __popc(avail_mask);
    // rank of this way among the available ones by (tick, way)
    int rank = 0;
    for (int l = 0; l < 32; ++l) {
      const int32_t t = __shfl_sync(0xffffffffu, tick, l);
      if (((avail_mask >> l) & 1u) && (t < tick || (t == tick && l < lane))) ++rank;
    }
    if (avail && rank < count) {
      const int64_t u = u_sorted[first + rank];
      const int64_t old = T.tags[slot];
      move[u] = (old >= 0 && T.dirty[slot]) ? old : -1;
      T.tags[slot] = uniq[u];
      T.ticks[slot] = now;
      T.dirty[slot] = train;
      slot_of[u] = slot;
    }
    // the misses the set cannot take this step: spill slot of their unique index
    for (int64_t i = n_avail + lane; i < count; i += 32) {
      const int64_t u = u_sorted[first + i];
      const int64_t sp = T.n_sets * 32 + u;
      T.tags[sp] = uniq[u];
      T.dirty[sp] = train;
      slot_of[u] = sp;
      move[u] = -1;
    }
    if (lane == 0) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[1]),
                static_cast<unsigned long long>(count));
      if (count > n_avail)
        atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[2]),
                  static_cast<unsigned long long>(count - n_avail));
    }
  }
}

// 6. fill: write back the evicted dirty row, then load the new one; advances the tick word
__global__ void __launch_bounds__(kCacheThreads)
    cache_fill_kernel(const __grid_constant__ CacheTable T, const int64_t* __restrict__ n_unique,
                      int64_t cap, const int64_t* __restrict__ uniq,
                      const int64_t* __restrict__ slot_of, const int64_t* __restrict__ move) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kCacheWarps;
  const int64_t nu = *n_unique;
  if (blockIdx.x == 0 && threadIdx.x == 0) *T.tick_word += 1;  // no other thread reads it here
  for (int64_t u = warp; u < nu && u < cap; u += n_warps) {
    const int64_t mv = move[u];
    if (mv == -2) continue;
    const int64_t slot = slot_of[u];
    if (mv >= 0) {
      move_row(T, slot, mv, true, lane);
      if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[3]), 1ull);
    }
    __syncwarp();
    move_row(T, slot, uniq[u], false, lane);
  }
}

// 7. remap: out[i] = slot of the row of id i, -1 when the id is outside the shard
template <typename IdT>
__global__ void __launch_bounds__(kCacheThreads)
    cache_remap_kernel(const CacheRemap* __restrict__ inputs, int n_inputs,
                       const int64_t* __restrict__ uniq, const int64_t* __restrict__ n_unique,
                       const int64_t* __restrict__ slot_of, int64_t rows, IdT* __restrict__ out) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kCacheThreads;
  const int64_t nu = *n_unique;
  for (int f = 0; f < n_inputs; ++f) {
    const CacheRemap R = inputs[f];
    const IdT* ids = reinterpret_cast<const IdT*>(R.ids);
    for (int64_t i = tid; i < R.n; i += stride) {
      const int64_t id = static_cast<int64_t>(ids[i]) + R.id_shift;
      int64_t slot = -1;
      if (static_cast<uint64_t>(id) < static_cast<uint64_t>(R.sub_rows)) {
        const int64_t key = R.row_base + id;
        int64_t lo = 0, hi = nu;  // first unique row >= key
        while (lo < hi) {
          const int64_t mid = (lo + hi) >> 1;
          if (uniq[mid] < key) lo = mid + 1;
          else hi = mid;
        }
        if (lo < nu && uniq[lo] == key && key < rows) slot = slot_of[lo];
      }
      out[R.out_off + i] = static_cast<IdT>(slot);
    }
  }
}

// every dirty slot (sets and spill region) -> host, dirty bits cleared; tags stay
__global__ void __launch_bounds__(kCacheThreads)
    cache_flush_kernel(const __grid_constant__ CacheTable T) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCacheThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kCacheWarps;
  const int64_t n_slots = T.n_sets * 32 + T.n_spill;
  for (int64_t slot = warp; slot < n_slots; slot += n_warps) {
    const int64_t row = T.tags[slot];
    if (row < 0 || !T.dirty[slot]) continue;
    move_row(T, slot, row, true, lane);
    __syncwarp();
    if (lane == 0) {
      T.dirty[slot] = 0;
      atomicAdd(reinterpret_cast<unsigned long long*>(&T.stats[3]), 1ull);
    }
  }
}

int warp_grid(int64_t n_warp_items, int sm_count) {
  int64_t blocks = (n_warp_items + kCacheWarps - 1) / kCacheWarps;
  const int64_t cap = static_cast<int64_t>(sm_count) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

}  // namespace

void launch_cache_spill_writeback(const CacheTable& T, int sm_count, cudaStream_t stream) {
  if (T.n_spill <= 0) return;
  cache_spill_writeback_kernel<<<warp_grid(T.n_spill, sm_count), kCacheThreads, 0, stream>>>(T);
}

void launch_cache_probe(const CacheTable& T, const int64_t* sorted_keys, const int64_t* seg_start,
                        const int64_t* n_unique, int64_t cap, bool train, int64_t* uniq,
                        uint32_t* miss_set, uint32_t* miss_item, int64_t* slot_of, int64_t* move,
                        int sm_count, cudaStream_t stream) {
  if (cap <= 0) return;
  cache_probe_kernel<<<warp_grid(cap, sm_count), kCacheThreads, 0, stream>>>(
      T, sorted_keys, seg_start, n_unique, cap, train ? 1 : 0, uniq, miss_set, miss_item, slot_of,
      move);
}

void launch_cache_assign(const CacheTable& T, const int64_t* set_sorted, const uint32_t* u_sorted,
                         const int64_t* seg, const int64_t* n_seg, int64_t cap, bool train,
                         const int64_t* uniq, int64_t* slot_of, int64_t* move, int sm_count,
                         cudaStream_t stream) {
  if (cap <= 0) return;
  cache_assign_kernel<<<warp_grid(cap, sm_count), kCacheThreads, 0, stream>>>(
      T, set_sorted, u_sorted, seg, n_seg, cap, train ? 1 : 0, uniq, slot_of, move);
}

void launch_cache_fill(const CacheTable& T, const int64_t* n_unique, int64_t cap,
                       const int64_t* uniq, const int64_t* slot_of, const int64_t* move,
                       int sm_count, cudaStream_t stream) {
  cache_fill_kernel<<<warp_grid(cap, sm_count), kCacheThreads, 0, stream>>>(T, n_unique, cap, uniq,
                                                                            slot_of, move);
}

void launch_cache_remap(const CacheRemap* inputs, int n_inputs, int64_t max_n,
                        const int64_t* uniq, const int64_t* n_unique, const int64_t* slot_of,
                        int64_t rows, bool ids64, void* out, int sm_count, cudaStream_t stream) {
  if (n_inputs <= 0 || max_n <= 0) return;
  int64_t blocks = (max_n + kCacheThreads - 1) / kCacheThreads;
  if (blocks > static_cast<int64_t>(sm_count) * 8) blocks = static_cast<int64_t>(sm_count) * 8;
  const int grid = static_cast<int>(blocks < 1 ? 1 : blocks);
  if (ids64)
    cache_remap_kernel<int64_t><<<grid, kCacheThreads, 0, stream>>>(
        inputs, n_inputs, uniq, n_unique, slot_of, rows, static_cast<int64_t*>(out));
  else
    cache_remap_kernel<int32_t><<<grid, kCacheThreads, 0, stream>>>(
        inputs, n_inputs, uniq, n_unique, slot_of, rows, static_cast<int32_t*>(out));
}

void launch_cache_flush(const CacheTable& T, int sm_count, cudaStream_t stream) {
  const int64_t n = T.n_sets * 32 + T.n_spill;
  if (n <= 0) return;
  cache_flush_kernel<<<warp_grid(n, sm_count), kCacheThreads, 0, stream>>>(T);
}

}  // namespace de
