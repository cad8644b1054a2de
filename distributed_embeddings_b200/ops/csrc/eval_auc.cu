// Exact ROC AUC of the DLRM evaluation (utils/metrics.py, ExactAUC), in integers.
//
// A prediction p in [0, 1] (fp32) with label y is stored as the 31-bit key
//   key = (bits(p) << 1) | (y > 0.5)
// bits(p) is monotone in p on [0, 1] and at most 0x3F800000, so sorting the keys
// (radix_sort_keys32, end_bit 31) orders the samples by score, negatives before positives within
// one score.  Over the sorted keys, with NP(i) = negatives at positions before i:
//   U2 = sum over positives j of (2 #{neg: p < p_j} + #{neg: p == p_j})
//      = sum over positives i of (NP(i) + NP(a_i))
// where a_i is the first position of i's score run: NP(i) counts the negatives of lower or equal
// score (equal ones sort before i), NP(a_i) those of lower score.  This is the familiar
// 2 * sum NP(i) - sum over runs of pos_run * neg_run, with the per-run correction folded into
// NP(a_i).  NP is a block scan of the negative flags plus tile prefixes; NP(a_i) is carried
// forward from each score-run head by a max-scan (NP never decreases).  Three kernels:
//   auc_tile_kernel  per tile: its negatives, and NP within the tile at its last run head
//   auc_scan_kernel  one block over the tiles: tile prefixes of NP and of the run-head carry; P, N
//   auc_u2_kernel    per tile: every positive's term, one uint64 atomic per block
// Integer atomics only: the result does not depend on the order of the blocks.
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "de_b200.h"

namespace de {
namespace {

constexpr int kAppendThreads = 256;
constexpr int kCountThreads = 256;
constexpr int kPerThread = 16;  // consecutive keys per thread
constexpr int kCountTile = kCountThreads * kPerThread;
constexpr int kScanThreads = 1024;

// Rows below *n_valid: key of (probs[i], labels[i]) -> keys[state[0] + i].  Every block reads the
// stored count before it takes a ticket; the last block to take one advances the count (or the
// dropped rows when the rows would pass `capacity`: then nothing is written) and clears the ticket,
// so the kernel replays inside a CUDA graph with all offsets on the device.
__global__ void __launch_bounds__(kAppendThreads)
    auc_append_kernel(const float* __restrict__ probs, const float* __restrict__ labels,
                      int64_t batch, const int64_t* __restrict__ n_valid,
                      uint32_t* __restrict__ keys, int64_t capacity,
                      unsigned long long* __restrict__ state) {
  __shared__ unsigned s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  int64_t nv = *n_valid;
  nv = nv < 0 ? 0 : (nv > batch ? batch : nv);
  const int64_t base = static_cast<int64_t>(*reinterpret_cast<volatile unsigned long long*>(state));
  const bool fits = base + nv <= capacity;
  unsigned bad = 0;
  if (fits) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
      const float p = probs[i];
      if (p >= 0.f && p <= 1.f) {
        // & 0x7fffffff: -0.0 is stored as 0.0, the value it equals
        keys[base + i] = ((__float_as_uint(p) & 0x7fffffffu) << 1) | (labels[i] > 0.5f ? 1u : 0u);
      } else {
        ++bad;  // NaN or out of range: not encoded, the result raises
      }
    }
  }
  bad = __reduce_add_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(&s_bad, bad);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_bad) atomicAdd(state + 2, static_cast<unsigned long long>(s_bad));
    __threadfence();
    if (atomicAdd(state + 3, 1ull) == gridDim.x - 1) {
      if (fits)
        state[0] = static_cast<unsigned long long>(base + nv);
      else
        state[1] += static_cast<unsigned long long>(nv);
      state[3] = 0;
    }
  }
}

// Exclusive scan of one value per thread over the block with an associative `op` and its
// identity; `total` receives the block-wide result.  `buf` holds 33 words.
template <typename T, typename Op>
__device__ __forceinline__ T block_exclusive(T v, T identity, Op op, T* buf, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  T incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = op(incl, t);
  }
  T excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = identity;
  if (lane == 31) buf[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    T s = lane < n_warps ? buf[lane] : identity;
    T si = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      T t = __shfl_up_sync(0xffffffffu, si, d);
      if (lane >= d) si = op(si, t);
    }
    T se = __shfl_up_sync(0xffffffffu, si, 1);
    if (lane < n_warps) buf[lane] = lane == 0 ? identity : se;  // exclusive warp prefix
    if (lane == 31) buf[32] = si;                               // block total
  }
  __syncthreads();
  const T r = op(buf[warp], excl);
  total = buf[32];
  __syncthreads();  // buf may be reused by the caller's next scan
  return r;
}

struct Add {
  template <typename T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct Max {
  template <typename T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a > b ? a : b; }
};

// The kPerThread keys of thread `threadIdx.x` in tile `blockIdx.x` (positions >= n read as 0 and
// are excluded by the callers), the key before them (all ones at position 0: a run head), the
// chunk's negatives and the negatives of the chunk before its last score-run head (-1: none).
struct Chunk {
  uint32_t k[kPerThread];
  int64_t i0;
  uint32_t prev;
  uint32_t neg;
  int last_head;
};

__device__ __forceinline__ void load_chunk(const uint32_t* __restrict__ keys, int64_t n,
                                           Chunk& c) {
  c.i0 = static_cast<int64_t>(blockIdx.x) * kCountTile + threadIdx.x * kPerThread;
  if (c.i0 + kPerThread <= n) {
    const uint4* src = reinterpret_cast<const uint4*>(keys + c.i0);
#pragma unroll
    for (int v = 0; v < kPerThread / 4; ++v) {
      const uint4 q = src[v];
      c.k[4 * v] = q.x;
      c.k[4 * v + 1] = q.y;
      c.k[4 * v + 2] = q.z;
      c.k[4 * v + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) c.k[j] = c.i0 + j < n ? keys[c.i0 + j] : 0u;
  }
  c.prev = c.i0 > 0 && c.i0 <= n ? keys[c.i0 - 1] : 0xffffffffu;
  c.neg = 0;
  c.last_head = -1;
  uint32_t prev = c.prev;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    if (c.i0 + j < n) {
      if ((c.k[j] >> 1) != (prev >> 1)) c.last_head = static_cast<int>(c.neg);
      c.neg += (c.k[j] & 1u) ^ 1u;
    }
    prev = c.k[j];
  }
}

__global__ void __launch_bounds__(kCountThreads)
    auc_tile_kernel(const uint32_t* __restrict__ keys, int64_t n, uint32_t* __restrict__ tile_neg,
                    int* __restrict__ tile_head) {
  __shared__ uint32_t s_sum[33];
  __shared__ int s_max[33];
  Chunk c;
  load_chunk(keys, n, c);
  uint32_t total;
  const uint32_t before = block_exclusive<uint32_t>(c.neg, 0u, Add(), s_sum, total);
  const int h = c.last_head >= 0 ? static_cast<int>(before) + c.last_head : -1;
  int last;
  block_exclusive<int>(h, -1, Max(), s_max, last);
  if (threadIdx.x == 0) {
    tile_neg[blockIdx.x] = total;
    tile_head[blockIdx.x] = last;
  }
}

// one block: tile_np[t] = negatives before tile t, tile_rs[t] = NP at the last score-run head
// before tile t (0 for tile 0); out = [P, N, 0]
__global__ void __launch_bounds__(kScanThreads)
    auc_scan_kernel(const uint32_t* __restrict__ tile_neg, const int* __restrict__ tile_head,
                    int64_t n_tiles, int64_t n, unsigned long long* __restrict__ tile_np,
                    unsigned long long* __restrict__ tile_rs, unsigned long long* __restrict__ out) {
  __shared__ unsigned long long buf[33];
  unsigned long long carry_np = 0, carry_rs = 0;
  for (int64_t c0 = 0; c0 < n_tiles; c0 += kScanThreads) {
    const int64_t t = c0 + threadIdx.x;
    const bool in = t < n_tiles;
    unsigned long long sum, top;
    const unsigned long long np =
        carry_np + block_exclusive<unsigned long long>(in ? tile_neg[t] : 0ull, 0ull, Add(), buf,
                                                       sum);
    const int h = in ? tile_head[t] : -1;
    const unsigned long long hv = h >= 0 ? np + static_cast<unsigned long long>(h) : 0ull;
    const unsigned long long rs = Max()(carry_rs, block_exclusive<unsigned long long>(
                                                      hv, 0ull, Max(), buf, top));
    if (in) {
      tile_np[t] = np;
      tile_rs[t] = rs;
    }
    carry_np += sum;
    carry_rs = Max()(carry_rs, top);
  }
  if (threadIdx.x == 0) {
    out[0] = static_cast<unsigned long long>(n) - carry_np;
    out[1] = carry_np;
    out[2] = 0;
  }
}

__global__ void __launch_bounds__(kCountThreads)
    auc_u2_kernel(const uint32_t* __restrict__ keys, int64_t n,
                  const unsigned long long* __restrict__ tile_np,
                  const unsigned long long* __restrict__ tile_rs,
                  unsigned long long* __restrict__ out) {
  __shared__ unsigned long long buf[33];
  Chunk c;
  load_chunk(keys, n, c);
  unsigned long long unused;
  unsigned long long np =
      tile_np[blockIdx.x] +
      block_exclusive<unsigned long long>(c.neg, 0ull, Add(), buf, unused);
  const unsigned long long hv =
      c.last_head >= 0 ? np + static_cast<unsigned long long>(c.last_head) : 0ull;
  unsigned long long rs =
      Max()(tile_rs[blockIdx.x], block_exclusive<unsigned long long>(hv, 0ull, Max(), buf, unused));
  unsigned long long acc = 0;
  uint32_t prev = c.prev;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    if (c.i0 + j < n) {
      if ((c.k[j] >> 1) != (prev >> 1)) rs = np;
      if (c.k[j] & 1u)
        acc += np + rs;
      else
        ++np;
    }
    prev = c.k[j];
  }
  unsigned long long block_acc;
  block_exclusive<unsigned long long>(acc, 0ull, Add(), buf, block_acc);
  if (threadIdx.x == 0 && block_acc) atomicAdd(out + 2, block_acc);
}

inline int64_t count_tiles(int64_t n) { return (n + kCountTile - 1) / kCountTile; }
inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

}  // namespace

void launch_auc_append(const float* probs, const float* labels, int64_t batch,
                       const int64_t* n_valid, uint32_t* keys, int64_t capacity, int64_t* state,
                       int sm_count, cudaStream_t stream) {
  int64_t blocks = (batch + kAppendThreads - 1) / kAppendThreads;
  const int64_t cap = static_cast<int64_t>(sm_count) * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  auc_append_kernel<<<static_cast<unsigned>(blocks), kAppendThreads, 0, stream>>>(
      probs, labels, batch, n_valid, keys, capacity,
      reinterpret_cast<unsigned long long*>(state));
}

// tile_neg, tile_head (4 bytes each), tile_np, tile_rs (8 bytes each) per tile of 4096 keys
size_t auc_count_temp_bytes(int64_t n) {
  const size_t t = static_cast<size_t>(count_tiles(n));
  return 2 * align256(t * 4) + 2 * align256(t * 8);
}

void launch_auc_count(void* temp, const uint32_t* sorted_keys, int64_t n, int64_t* out,
                      cudaStream_t stream) {
  if (n <= 0) {
    cudaMemsetAsync(out, 0, 3 * sizeof(int64_t), stream);
    return;
  }
  const int64_t n_tiles = count_tiles(n);
  char* p = static_cast<char*>(temp);
  uint32_t* tile_neg = reinterpret_cast<uint32_t*>(p);
  p += align256(static_cast<size_t>(n_tiles) * 4);
  int* tile_head = reinterpret_cast<int*>(p);
  p += align256(static_cast<size_t>(n_tiles) * 4);
  unsigned long long* tile_np = reinterpret_cast<unsigned long long*>(p);
  p += align256(static_cast<size_t>(n_tiles) * 8);
  unsigned long long* tile_rs = reinterpret_cast<unsigned long long*>(p);
  unsigned long long* o = reinterpret_cast<unsigned long long*>(out);
  auc_tile_kernel<<<static_cast<unsigned>(n_tiles), kCountThreads, 0, stream>>>(
      sorted_keys, n, tile_neg, tile_head);
  auc_scan_kernel<<<1, kScanThreads, 0, stream>>>(tile_neg, tile_head, n_tiles, n, tile_np,
                                                  tile_rs, o);
  auc_u2_kernel<<<static_cast<unsigned>(n_tiles), kCountThreads, 0, stream>>>(
      sorted_keys, n, tile_np, tile_rs, o);
}

}  // namespace de
