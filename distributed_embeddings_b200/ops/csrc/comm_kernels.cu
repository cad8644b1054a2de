// NVLink / NVSwitch communication kernels for sm_90a: flag barrier over peer-mapped signal pads
// and the dense-gradient all-reduce (the data-parallel half of hybrid parallelism) as a single
// kernel: reduce-scatter + all-gather over peer memory, fused with the 1/world scale and the
// bf16/fp32 handling, either with plain P2P loads/stores or with NVSwitch multicast
// (multimem.ld_reduce / multimem.st -> in-switch reduction).
//
// Replaces Horovod's allreduce / barrier use (reference dist_model_parallel.py:1260, 985).
#include <algorithm>

#include "common.cuh"

namespace de {

namespace {

// ----------------------------------------------------------------------------- barrier
// grid = 1 block.  Thread t < world signals peer t and waits for peer t.
__global__ void barrier_kernel(const __grid_constant__ PeerPtrs flags, uint32_t* epoch_p, int rank,
                               int world, int channel, unsigned long long timeout_cycles,
                               int* error_flag) {
  const uint32_t epoch = *epoch_p + 1;
  const int t = threadIdx.x;
  if (t < world) {
    __threadfence_system();
    st_release_sys(flag_slot(flags.p[t], channel, rank), epoch);
    if (!wait_flag_ge(flag_slot(flags.p[rank], channel, t), epoch, timeout_cycles))
      peer_timeout_trap(error_flag, t);  // never continue (or advance the epoch) past a lost peer
  }
  __syncthreads();
  if (t == 0) *epoch_p = epoch;
}

// Multi-block entry barrier: block 0 signals, every block waits (flags are local memory).
__device__ __forceinline__ void grid_peer_barrier_enter(const PeerPtrs& flags, uint32_t epoch,
                                                        int rank, int world, int channel,
                                                        unsigned long long timeout_cycles,
                                                        int* error_flag) {
  const int t = threadIdx.x;
  if (t < world) {
    if (blockIdx.x == 0) {
      __threadfence_system();
      st_release_sys(flag_slot(flags.p[t], channel, rank), epoch);
    }
    if (!wait_flag_ge(flag_slot(flags.p[rank], channel, t), epoch, timeout_cycles))
      peer_timeout_trap(error_flag, t);  // never continue (or advance the epoch) past a lost peer
  }
  __syncthreads();
}

// Multi-block exit barrier: the last block to finish signals the peers and waits for them, so
// kernel completion implies every rank's writes into this rank's buffer have landed.
__device__ __forceinline__ void grid_peer_barrier_exit(const PeerPtrs& flags, uint32_t epoch,
                                                       uint32_t* block_counter, uint32_t* epoch_p,
                                                       int rank, int world, int channel,
                                                       unsigned long long timeout_cycles,
                                                       int* error_flag) {
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t done = atomicAdd(block_counter, 1u);
    last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  const int t = threadIdx.x;
  if (t < world) {
    __threadfence_system();
    st_release_sys(flag_slot(flags.p[t], channel, rank), epoch);
    if (!wait_flag_ge(flag_slot(flags.p[rank], channel, t), epoch, timeout_cycles))
      peer_timeout_trap(error_flag, t);  // never continue (or advance the epoch) past a lost peer
  }
  __syncthreads();
  if (t == 0) {
    *block_counter = 0;
    *epoch_p = epoch;
  }
}

// ----------------------------------------------------------------------------- all-reduce
// Rank r owns the r-th slice: it sums the slice over all peers (P2P loads), scales, and stores
// the result into every peer's buffer (P2P stores).  16-byte accesses; n_vec = elements / VEC.
__device__ __forceinline__ void acc_f32(float (&a)[4], const uint4& v) {
  a[0] += __uint_as_float(v.x);
  a[1] += __uint_as_float(v.y);
  a[2] += __uint_as_float(v.z);
  a[3] += __uint_as_float(v.w);
}
__device__ __forceinline__ void acc_bf16(float (&a)[8], const uint4& v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[i]);
    float2 f = __bfloat1622float2(h);
    a[2 * i] += f.x;
    a[2 * i + 1] += f.y;
  }
}

template <bool BF16>
__global__ void __launch_bounds__(512)
allreduce_p2p_kernel(const __grid_constant__ PeerPtrs bufs, const __grid_constant__ PeerPtrs flags,
                     uint32_t* epoch_p, uint32_t* block_counter, int rank, int world,
                     int64_t n_vec16, float scale, int channel, unsigned long long timeout_cycles,
                     int* error_flag) {
  const uint32_t epoch = *epoch_p + 1;
  grid_peer_barrier_enter(flags, epoch, rank, world, channel, timeout_cycles, error_flag);

  const int64_t per = (n_vec16 + world - 1) / world;
  const int64_t lo = per * rank;
  const int64_t hi = min(n_vec16, lo + per);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = lo + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < hi;
       i += stride) {
    uint4 v[kMaxPeers];
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) {
      if (p < world) {
        const int q = (rank + p) % world;  // stagger peers
        v[p] = reinterpret_cast<const uint4*>(bufs.p[q])[i];
      }
    }
    uint4 o;
    if constexpr (BF16) {
      float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p)
        if (p < world) acc_bf16(a, v[p]);
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a[2 * j] * scale, a[2 * j + 1] * scale);
        w[j] = *reinterpret_cast<uint32_t*>(&h);
      }
      o = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
      float a[4] = {0, 0, 0, 0};
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p)
        if (p < world) acc_f32(a, v[p]);
      o = make_uint4(__float_as_uint(a[0] * scale), __float_as_uint(a[1] * scale),
                     __float_as_uint(a[2] * scale), __float_as_uint(a[3] * scale));
    }
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) {
      if (p < world) {
        const int q = (rank + p) % world;
        reinterpret_cast<uint4*>(bufs.p[q])[i] = o;
      }
    }
  }
  grid_peer_barrier_exit(flags, epoch + 1, block_counter, epoch_p, rank, world, channel,
                         timeout_cycles, error_flag);
}

// NVSwitch multicast variant: one multimem.ld_reduce pulls the switch-reduced 16 bytes, one
// multimem.st broadcasts the scaled result to every GPU.
template <bool BF16>
__global__ void __launch_bounds__(512)
allreduce_multimem_kernel(void* mc_ptr, const __grid_constant__ PeerPtrs flags, uint32_t* epoch_p,
                          uint32_t* block_counter, int rank, int world, int64_t n_vec16,
                          float scale, int channel, unsigned long long timeout_cycles,
                          int* error_flag) {
  const uint32_t epoch = *epoch_p + 1;
  grid_peer_barrier_enter(flags, epoch, rank, world, channel, timeout_cycles, error_flag);
  const int64_t per = (n_vec16 + world - 1) / world;
  const int64_t lo = per * rank;
  const int64_t hi = min(n_vec16, lo + per);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  uint4* mc = reinterpret_cast<uint4*>(mc_ptr);
  for (int64_t i = lo + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < hi;
       i += stride) {
    uint4 o;
    if constexpr (BF16) {
      uint32_t x0, x1, x2, x3;
      asm volatile(
          "multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
          : "=r"(x0), "=r"(x1), "=r"(x2), "=r"(x3)
          : "l"(mc + i)
          : "memory");
      uint32_t w[4] = {x0, x1, x2, x3};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&w[j]);
        float2 f = __bfloat1622float2(h);
        h = __floats2bfloat162_rn(f.x * scale, f.y * scale);
        w[j] = *reinterpret_cast<uint32_t*>(&h);
      }
      o = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
      float a, b, c, d;
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(a), "=f"(b), "=f"(c), "=f"(d)
                   : "l"(mc + i)
                   : "memory");
      o = make_uint4(__float_as_uint(a * scale), __float_as_uint(b * scale),
                     __float_as_uint(c * scale), __float_as_uint(d * scale));
    }
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + i),
                 "f"(__uint_as_float(o.x)), "f"(__uint_as_float(o.y)), "f"(__uint_as_float(o.z)),
                 "f"(__uint_as_float(o.w))
                 : "memory");
  }
  grid_peer_barrier_exit(flags, epoch + 1, block_counter, epoch_p, rank, world, channel,
                         timeout_cycles, error_flag);
}

// ----------------------------------------------------------------------------- P2P store probe
// Micro-benchmark of kernel-issued stores into peer memory (tools/bench_p2p_store.py): row r of a
// contiguous local buffer goes to dst + r * dst_stride.  VEC bytes per lane; a warp instruction
// covers 32 * VEC contiguous bytes of one row (or several whole rows when the row is shorter),
// which is exactly how the lookup / gradient-push kernels emit their rows.
template <typename V>
__global__ void __launch_bounds__(1024)
p2p_store_bench_kernel(const char* __restrict__ src, char* __restrict__ dst, int64_t n_rows,
                       int row_bytes, int64_t dst_stride, int unroll) {
  constexpr int VB = sizeof(V);
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int lanes_per_row = row_bytes / VB;  // <= 32 handled as several rows per instruction
  if (lanes_per_row >= 32) {
    const int chunks = lanes_per_row / 32;
    for (int64_t r = warp; r < n_rows; r += n_warps) {
      const V* sp = reinterpret_cast<const V*>(src + r * row_bytes);
      V* dp = reinterpret_cast<V*>(dst + r * dst_stride);
      for (int c = 0; c < chunks; ++c) dp[c * 32 + lane] = sp[c * 32 + lane];
    }
  } else {
    const int rpi = 32 / lanes_per_row;  // rows per instruction
    const int sub = lane / lanes_per_row, li = lane - sub * lanes_per_row;
    for (int64_t r0 = warp * rpi * unroll; r0 < n_rows; r0 += n_warps * rpi * unroll) {
      V v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t r = r0 + u * rpi + sub;
        if (u < unroll && r < n_rows) v[u] = reinterpret_cast<const V*>(src + r * row_bytes)[li];
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t r = r0 + u * rpi + sub;
        if (u < unroll && r < n_rows) reinterpret_cast<V*>(dst + r * dst_stride)[li] = v[u];
      }
    }
  }
}

// ----------------------------------------------------------------------------- signalling only
__global__ void sync_only_kernel(const __grid_constant__ SyncArgs sync) {
  sync_head(sync);
  sync_tail(sync);
}

// ----------------------------------------------------------------------------- index push
// Push-style all-to-all of index segments: segment j copies n elements of the local staging
// buffer into the id buffer of the rank that owns the feature (fire-and-forget NVLink stores;
// the reference's 'inp_dp_to_mp' hvd.alltoall, dist_model_parallel.py:211).  The head waits
// until every owner has consumed the ids of the previous step (wait_abs on the "consumed"
// channel), the tail tells the owners that their ids are complete.
template <typename T>
__global__ void __launch_bounds__(256)
push_segments_kernel(const int64_t* __restrict__ segs, int n_seg, const T* __restrict__ src,
                     const __grid_constant__ PeerPtrs dst, int blocks_per_seg,
                     const __grid_constant__ SyncArgs sync) {
  sync_head(sync);
  const int j = blockIdx.x / blocks_per_seg;
  const int bj = blockIdx.x - j * blocks_per_seg;
  if (j < n_seg) {
    const int64_t* sg = segs + 4 * static_cast<int64_t>(j);
    const T* sp = src + sg[1];
    T* dp = reinterpret_cast<T*>(dst.p[sg[0]]) + sg[2];
    const int64_t n = sg[3];
    constexpr int kPer16 = 16 / sizeof(T);
    const int64_t stride = static_cast<int64_t>(blocks_per_seg) * blockDim.x;
    const int64_t t0 = static_cast<int64_t>(bj) * blockDim.x + threadIdx.x;
    if (((reinterpret_cast<uintptr_t>(sp) | reinterpret_cast<uintptr_t>(dp)) & 15) == 0) {
      const int64_t n16 = n / kPer16;
      for (int64_t i = t0; i < n16; i += stride)
        reinterpret_cast<uint4*>(dp)[i] = reinterpret_cast<const uint4*>(sp)[i];
      for (int64_t i = n16 * kPer16 + t0; i < n; i += stride) dp[i] = sp[i];
    } else {
      for (int64_t i = t0; i < n; i += stride) dp[i] = sp[i];
    }
  }
  sync_tail(sync);
}

// ----------------------------------------------------------------------------- gradient push
// The gradient all-to-all (Horovod's alltoall gradient in the reference) as a push: block row
// tiles x route pieces; every piece of a local gradient row is cast to the wire dtype and
// stored into the receive buffer of the rank that owns the table (slice).  16-byte stores when
// the piece allows it.
template <typename S, typename D>
__global__ void __launch_bounds__(256)
push_grad_kernel(const GradRoute* __restrict__ routes, int n_routes, const S* __restrict__ src,
                 int64_t src_stride, int64_t rows, float scale,
                 const __grid_constant__ SyncArgs sync) {
  sync_head(sync);
  constexpr int kRowsPerTile = 8;
  const int64_t n_row_tiles = (rows + kRowsPerTile - 1) / kRowsPerTile;
  const int64_t total = n_row_tiles * n_routes;
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int r = static_cast<int>(t % n_routes);
    const int64_t row0 = (t / n_routes) * kRowsPerTile;
    const GradRoute R = routes[r];
    D* dst = reinterpret_cast<D*>(R.dst);
    const int64_t left = rows - row0;
    const int nr = left < kRowsPerTile ? static_cast<int>(left) : kRowsPerTile;
    constexpr int kVec = 16 / sizeof(D);  // elements per 16-byte store
    const bool vec = (R.width % kVec == 0) && (R.dst_col % kVec == 0) &&
                     (R.dst_stride % kVec == 0) && (R.src_col % 4 == 0) && (src_stride % 4 == 0) &&
                     ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
    if (vec) {
      const int chunks = R.width / kVec;
      for (int c = threadIdx.x; c < nr * chunks; c += blockDim.x) {
        const int rr = c / chunks, ch = c - rr * chunks;
        const S* sp = src + (row0 + rr) * src_stride + R.src_col + ch * kVec;
        float v[kVec];
#pragma unroll
        for (int k = 0; k < kVec; ++k) v[k] = to_f32<S>(sp[k]) * scale;
        D* dp = dst + (row0 + rr) * R.dst_stride + R.dst_col + ch * kVec;
        if constexpr (sizeof(D) == 4) {
          *reinterpret_cast<float4*>(dp) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
          uint4 o;
          o.x = pack2<D>(v[0], v[1]);
          o.y = pack2<D>(v[2], v[3]);
          o.z = pack2<D>(v[4], v[5]);
          o.w = pack2<D>(v[6], v[7]);
          *reinterpret_cast<uint4*>(dp) = o;
        }
      }
    } else {
      for (int c = threadIdx.x; c < nr * R.width; c += blockDim.x) {
        const int rr = c / R.width, cc = c - rr * R.width;
        dst[(row0 + rr) * R.dst_stride + R.dst_col + cc] =
            from_f32<D>(to_f32<S>(src[(row0 + rr) * src_stride + R.src_col + cc]) * scale);
      }
    }
  }
  sync_tail(sync);
}

// ----------------------------------------------------------------------------- streamed push
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(512)
stream_push_kernel(const __grid_constant__ PushPlan plan, const uint32_t* __restrict__ counters,
                   int chunk_rows, int64_t rows, unsigned long long timeout, int* error_flag,
                   const __grid_constant__ SyncArgs sync) {
  const int64_t n_chunks = (rows + chunk_rows - 1) / chunk_rows;
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t n_thr = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const int64_t r0 = c * chunk_rows;
    const int64_t left = rows - r0;
    const uint32_t nr = static_cast<uint32_t>(left < chunk_rows ? left : chunk_rows);
    if (threadIdx.x == 0) {
      // the producer of this GPU counts finished rows per chunk (local memory: cheap to poll)
      const unsigned long long start = clock64();
      unsigned spins = 0;
      while (ld_acquire_gpu_u32(counters + c) < nr) {
        if ((++spins & 0x3ff) == 0 && timeout && (clock64() - start) > timeout)
          peer_timeout_trap(error_flag, sync.rank);
        __nanosleep(100);
      }
    }
    __syncthreads();
    for (int p = 0; p < plan.n; ++p) {
      const int64_t n16 = (static_cast<int64_t>(nr) * plan.row_bytes[p]) >> 4;
      const uint4* sp = reinterpret_cast<const uint4*>(static_cast<const char*>(plan.src[p]) +
                                                       r0 * plan.row_bytes[p]);
      uint4* dp = reinterpret_cast<uint4*>(static_cast<char*>(plan.dst[p]) +
                                           r0 * plan.row_bytes[p]);
      constexpr int kU = 4;
      int64_t i = tid;
      for (; i + (kU - 1) * n_thr < n16; i += kU * n_thr) {
        uint4 v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) v[u] = sp[i + u * n_thr];
#pragma unroll
        for (int u = 0; u < kU; ++u) dp[i + u * n_thr] = v[u];
      }
      for (; i < n16; i += n_thr) dp[i] = sp[i];
    }
  }
  sync_tail(sync);  // every staged row is on its way: "gradient ready" to the owners
}

// ----------------------------------------------------------------------------- row-slice sum
// Multi-hot row-sliced inputs: every rank pooled the ids it owns and stored its partial result
// in slot `rank` of the requester; the requester sums the W slots into its output row (the
// reference's reduce-scatter, dist_model_parallel.py:291-298, without the W-fold redundancy in
// the output direction).
template <typename OutT>
__global__ void __launch_bounds__(256)
rowslice_reduce_kernel(const float* __restrict__ partial, int world, int64_t rows,
                       int64_t part_stride, OutT* __restrict__ out, int64_t out_stride,
                       const int32_t* __restrict__ cols, int n_cols, int total_width) {
  const int64_t n = rows * total_width;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    const int64_t r = i / total_width;
    int c = static_cast<int>(i - r * total_width);
    // find the column group (few groups: linear scan)
    int j = 0, base = 0;
    while (j < n_cols - 1 && c >= base + cols[3 * j + 2]) {
      base += cols[3 * j + 2];
      ++j;
    }
    c -= base;
    float acc = 0.f;
    for (int s = 0; s < world; ++s)
      acc += partial[(static_cast<int64_t>(s) * rows + r) * part_stride + cols[3 * j] + c];
    out[r * out_stride + cols[3 * j + 1] + c] = from_f32<OutT>(acc);
  }
}

// Pull-style all-to-all of index segments: segment j copies n elements from peer src_rank's
// staging buffer into the local model-parallel id buffer (the reference's 'inp_dp_to_mp'
// hvd.alltoall, dist_model_parallel.py:211, as direct NVLink reads).
template <typename T>
__global__ void gather_segments_kernel(const int64_t* __restrict__ segs,
                                       const __grid_constant__ PeerPtrs src, T* __restrict__ dst) {
  const int64_t* sg = segs + 4 * static_cast<int64_t>(blockIdx.y);
  const T* sp = reinterpret_cast<const T*>(src.p[sg[0]]) + sg[1];
  T* dp = dst + sg[2];
  const int64_t n = sg[3];
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    dp[i] = sp[i];
}

// Double-buffered input staging for graph-replayed steps: copies the active staging slot
// (chosen by a device-resident flag, so one captured graph serves both slots) into the static
// input buffers.  All sizes are multiples of 16 bytes.
struct SelectSegs {
  const uint4* src[2][4];
  uint4* dst[4];
  int64_t n16[4];
  int count;
};
__global__ void select_copy_kernel(const __grid_constant__ SelectSegs segs,
                                   const int* __restrict__ slot_flag) {
  const int slot = (*slot_flag) & 1;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int s = 0; s < segs.count; ++s) {
    const uint4* src = segs.src[slot][s];
    uint4* dst = segs.dst[s];
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < segs.n16[s];
         i += stride)
      dst[i] = src[i];
  }
}

// Ragged index exchange over peer memory (replaces the reference's two hvd.alltoall calls for
// values + row lengths and the worker-major -> feature-major transpose, dist_model_parallel.py:
// 90-166).  Every requester stages values[cap] and row_splits[b+1] of a ragged feature in
// symmetric buffers; the owner pulls them from all sources and builds the global-batch CSR:
//   vals[item_off + base_s + j] = values_s[j],  goff[s*b + i] = base_s + splits_s[i],
// with base_s = sum of the earlier sources' nnz computed on the device (no host round trip).
// segs[j] = {src_val_off, dst_item_off, splits_off, goff_off}
template <typename T>
__global__ void gather_ragged_kernel(const int64_t* __restrict__ segs,
                                     const __grid_constant__ PeerPtrs src_vals,
                                     const __grid_constant__ PeerPtrs src_splits,
                                     T* __restrict__ dst_vals, int64_t* __restrict__ goff,
                                     int64_t b, int world) {
  const int64_t* sg = segs + 4 * static_cast<int64_t>(blockIdx.y);
  const int s = blockIdx.z;
  __shared__ int64_t s_base, s_nnz;
  if (threadIdx.x == 0) {
    int64_t base = 0;
    for (int q = 0; q < s; ++q)
      base += (reinterpret_cast<const int64_t*>(src_splits.p[q]) + sg[2])[b];
    s_base = base;
    s_nnz = (reinterpret_cast<const int64_t*>(src_splits.p[s]) + sg[2])[b];
  }
  __syncthreads();
  const int64_t base = s_base, nnz = s_nnz;
  const int64_t* sp = reinterpret_cast<const int64_t*>(src_splits.p[s]) + sg[2];
  const T* vals = reinterpret_cast<const T*>(src_vals.p[s]) + sg[0];
  T* dv = dst_vals + sg[1] + base;
  int64_t* go = goff + sg[3] + static_cast<int64_t>(s) * b;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t t0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (int64_t i = t0; i < nnz; i += stride) dv[i] = vals[i];
  for (int64_t i = t0; i < b; i += stride) go[i] = base + sp[i];
  if (s == world - 1 && t0 == 0) go[b] = base + nnz;
}

template <typename S, typename D>
__global__ void copy_cast_2d_kernel(const S* __restrict__ src, int64_t src_stride,
                                    D* __restrict__ dst, int64_t dst_stride, int64_t rows,
                                    int64_t cols, float scale) {
  const int64_t n = rows * cols;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    const int64_t r = i / cols, c = i - r * cols;
    dst[r * dst_stride + c] = from_f32<D>(to_f32<S>(src[r * src_stride + c]) * scale);
  }
}

}  // namespace

void launch_barrier(const PeerPtrs& flags, uint32_t* epoch, int rank, int world, int channel,
                    unsigned long long timeout_cycles, int* error_flag, cudaStream_t stream) {
  barrier_kernel<<<1, 32, 0, stream>>>(flags, epoch, rank, world, channel, timeout_cycles,
                                       error_flag);
}

// epoch[0] = epoch counter (advances by 2 per all-reduce), epoch[1] = block counter
void launch_allreduce(const PeerPtrs& bufs, const PeerPtrs& flags, uint32_t* epoch, int rank,
                      int world, int64_t n_elems, float scale, bool bf16, int channel,
                      unsigned long long timeout_cycles, int* error_flag, int sm_count,
                      cudaStream_t stream, int max_blocks) {
  const int64_t per16 = bf16 ? 8 : 4;
  const int64_t n_vec16 = (n_elems + per16 - 1) / per16;  // buffers are padded to 16 bytes
  const int threads = 512;
  int64_t blocks = ((n_vec16 + world - 1) / world + threads - 1) / threads;
  if (blocks > sm_count) blocks = sm_count;  // at most one wave: blocks spin on flags
  // an all-reduce that overlaps other kernels must leave most SMs to them: its blocks spin on
  // peer flags, and a spinning grid that fills the machine can starve the very kernels the
  // peers are waiting for
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  if (bf16)
    allreduce_p2p_kernel<true><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        bufs, flags, epoch, epoch + 1, rank, world, n_vec16, scale, channel, timeout_cycles,
        error_flag);
  else
    allreduce_p2p_kernel<false><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        bufs, flags, epoch, epoch + 1, rank, world, n_vec16, scale, channel, timeout_cycles,
        error_flag);
}

void launch_allreduce_multimem(void* mc_ptr, const PeerPtrs& flags, uint32_t* epoch, int rank,
                               int world, int64_t n_elems, float scale, bool bf16, int channel,
                               unsigned long long timeout_cycles, int* error_flag, int sm_count,
                               cudaStream_t stream, int max_blocks) {
  const int64_t per16 = bf16 ? 8 : 4;
  const int64_t n_vec16 = (n_elems + per16 - 1) / per16;
  const int threads = 512;
  int64_t blocks = ((n_vec16 + world - 1) / world + threads - 1) / threads;
  if (blocks > sm_count) blocks = sm_count;
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  if (bf16)
    allreduce_multimem_kernel<true><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        mc_ptr, flags, epoch, epoch + 1, rank, world, n_vec16, scale, channel, timeout_cycles,
        error_flag);
  else
    allreduce_multimem_kernel<false><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        mc_ptr, flags, epoch, epoch + 1, rank, world, n_vec16, scale, channel, timeout_cycles,
        error_flag);
}

void launch_select_copy(const void* const* src0, const void* const* src1, void* const* dst,
                        const int64_t* nbytes, int count, const int* slot_flag, int sm_count,
                        cudaStream_t stream) {
  SelectSegs segs;
  segs.count = count > 4 ? 4 : count;
  int64_t total = 0;
  for (int i = 0; i < segs.count; ++i) {
    segs.src[0][i] = reinterpret_cast<const uint4*>(src0[i]);
    segs.src[1][i] = reinterpret_cast<const uint4*>(src1[i]);
    segs.dst[i] = reinterpret_cast<uint4*>(dst[i]);
    segs.n16[i] = nbytes[i] / 16;
    total += segs.n16[i];
  }
  if (total == 0) return;
  int64_t blocks = (total + 255) / 256;
  if (blocks > sm_count * 4) blocks = sm_count * 4;
  select_copy_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(segs, slot_flag);
}

void launch_gather_ragged(const int64_t* segs, int n_seg, const PeerPtrs& src_vals,
                          const PeerPtrs& src_splits, void* dst_vals, int64_t* goff, int64_t b,
                          int world, int elem_bytes, int64_t max_cap, cudaStream_t stream) {
  if (n_seg <= 0) return;
  int64_t bx = (max_cap + 1023) / 1024;
  if (bx > 32) bx = 32;
  if (bx < 1) bx = 1;
  dim3 grid(static_cast<unsigned>(bx), static_cast<unsigned>(n_seg), static_cast<unsigned>(world));
  if (elem_bytes == 8)
    gather_ragged_kernel<int64_t><<<grid, 256, 0, stream>>>(
        segs, src_vals, src_splits, reinterpret_cast<int64_t*>(dst_vals), goff, b, world);
  else
    gather_ragged_kernel<int32_t><<<grid, 256, 0, stream>>>(
        segs, src_vals, src_splits, reinterpret_cast<int32_t*>(dst_vals), goff, b, world);
}

void launch_gather_segments(const int64_t* segs, int n_seg, const PeerPtrs& src, void* dst,
                            int elem_bytes, int64_t max_seg_elems, cudaStream_t stream) {
  if (n_seg <= 0 || max_seg_elems <= 0) return;
  const int threads = 256;
  int64_t bx = (max_seg_elems + threads * 4 - 1) / (threads * 4);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  dim3 grid(static_cast<unsigned>(bx), static_cast<unsigned>(n_seg));
  if (elem_bytes == 8)
    gather_segments_kernel<int64_t><<<grid, threads, 0, stream>>>(segs, src,
                                                                  reinterpret_cast<int64_t*>(dst));
  else
    gather_segments_kernel<int32_t><<<grid, threads, 0, stream>>>(segs, src,
                                                                  reinterpret_cast<int32_t*>(dst));
}

// 16-byte fast path: same dtype, unit scale, everything 16-byte aligned
__global__ void copy_2d_vec16_kernel(const uint4* __restrict__ src, int64_t src_stride16,
                                     uint4* __restrict__ dst, int64_t dst_stride16, int64_t rows,
                                     int64_t cols16) {
  const int64_t n = rows * cols16;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    const int64_t r = i / cols16, c = i - r * cols16;
    dst[r * dst_stride16 + c] = src[r * src_stride16 + c];
  }
}

void launch_copy_cast_2d(const void* src, int64_t src_stride, void* dst, int64_t dst_stride,
                         int64_t rows, int64_t cols, int src_dtype, int dst_dtype, float scale,
                         cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return;
  {
    const int64_t per16 = src_dtype == 0 ? 4 : 8;
    if (src_dtype == dst_dtype && scale == 1.0f && cols % per16 == 0 && src_stride % per16 == 0 &&
        dst_stride % per16 == 0 &&
        ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
      const int64_t n = rows * (cols / per16);
      int64_t blocks = (n + 255) / 256;
      if (blocks > kGridCapSms * 16) blocks = kGridCapSms * 16;
      copy_2d_vec16_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
          reinterpret_cast<const uint4*>(src), src_stride / per16, reinterpret_cast<uint4*>(dst),
          dst_stride / per16, rows, cols / per16);
      return;
    }
  }
  const int threads = 256;
  int64_t blocks = (rows * cols + threads - 1) / threads;
  if (blocks > kGridCapSms * 8) blocks = kGridCapSms * 8;
  with_dtype(src_dtype, [&](auto src_t) {
    using S = typename decltype(src_t)::type;
    with_dtype(dst_dtype, [&](auto dst_t) {
      using D = typename decltype(dst_t)::type;
      copy_cast_2d_kernel<S, D><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
          reinterpret_cast<const S*>(src), src_stride, reinterpret_cast<D*>(dst), dst_stride, rows,
          cols, scale);
    });
  });
}

void launch_p2p_store_bench(const void* src, void* dst, int64_t n_rows, int row_bytes,
                            int vec_bytes, int64_t dst_stride, int unroll, int blocks, int threads,
                            cudaStream_t stream) {
  const char* s = static_cast<const char*>(src);
  char* d = static_cast<char*>(dst);
  if (vec_bytes == 16)
    p2p_store_bench_kernel<uint4><<<blocks, threads, 0, stream>>>(s, d, n_rows, row_bytes,
                                                                  dst_stride, unroll);
  else if (vec_bytes == 8)
    p2p_store_bench_kernel<uint2><<<blocks, threads, 0, stream>>>(s, d, n_rows, row_bytes,
                                                                  dst_stride, unroll);
  else
    p2p_store_bench_kernel<uint32_t><<<blocks, threads, 0, stream>>>(s, d, n_rows, row_bytes,
                                                                     dst_stride, unroll);
}

void launch_stream_push(const PushPlan& plan, const uint32_t* counters, int chunk_rows,
                        int64_t rows, unsigned long long timeout, int* error_flag, int blocks,
                        cudaStream_t stream, const SyncArgs& sync) {
  if (plan.n <= 0 || rows <= 0) {
    launch_sync_only(sync, stream);
    return;
  }
  stream_push_kernel<<<blocks, 512, 0, stream>>>(plan, counters, chunk_rows, rows, timeout,
                                                 error_flag, sync);
}

void launch_sync_only(const SyncArgs& sync, cudaStream_t stream) {
  if (sync.state == nullptr || (sync.wait_ch < 0 && sync.wait_abs_ch < 0 && sync.signal_ch < 0))
    return;
  sync_only_kernel<<<1, 32, 0, stream>>>(sync);
}

void launch_push_segments(const int64_t* segs, int n_seg, const void* src, const PeerPtrs& dst,
                          int elem_bytes, int64_t max_seg_elems, int sm_count,
                          cudaStream_t stream, const SyncArgs& sync) {
  if (n_seg <= 0 || max_seg_elems <= 0) {
    launch_sync_only(sync, stream);
    return;
  }
  // 16-byte copies, 4 per thread: enough blocks per segment to cover the longest one, but never
  // more than one wave (every block spins in sync_head until the peers are ready)
  const int64_t per_block = 256 * 4 * (16 / elem_bytes);
  int64_t bps = (max_seg_elems + per_block - 1) / per_block;
  const int64_t cap = std::max<int64_t>(1, (static_cast<int64_t>(sm_count) * 4) / n_seg);
  if (bps > cap) bps = cap;
  if (bps < 1) bps = 1;
  const unsigned grid = static_cast<unsigned>(bps * n_seg);
  if (elem_bytes == 8)
    push_segments_kernel<int64_t><<<grid, 256, 0, stream>>>(
        segs, n_seg, reinterpret_cast<const int64_t*>(src), dst, static_cast<int>(bps), sync);
  else
    push_segments_kernel<int32_t><<<grid, 256, 0, stream>>>(
        segs, n_seg, reinterpret_cast<const int32_t*>(src), dst, static_cast<int>(bps), sync);
}

void launch_push_grad(const GradRoute* routes, int n_routes, const void* src, int64_t src_stride,
                      int src_dtype, int dst_dtype, int64_t rows, float scale, int sm_count,
                      cudaStream_t stream, const SyncArgs& sync) {
  if (n_routes <= 0 || rows <= 0) {
    launch_sync_only(sync, stream);
    return;
  }
  const int64_t total = ((rows + 7) / 8) * n_routes;
  int64_t blocks = total;
  if (blocks > static_cast<int64_t>(sm_count) * 8) blocks = static_cast<int64_t>(sm_count) * 8;
  with_dtype(src_dtype, [&](auto src_t) {
    using S = typename decltype(src_t)::type;
    with_dtype(dst_dtype, [&](auto dst_t) {
      using D = typename decltype(dst_t)::type;
      push_grad_kernel<S, D><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
          routes, n_routes, reinterpret_cast<const S*>(src), src_stride, rows, scale, sync);
    });
  });
}

void launch_rowslice_reduce(const float* partial, int world, int64_t rows, int64_t part_stride,
                            void* out, int64_t out_stride, int out_dtype, const int32_t* cols,
                            int n_cols, cudaStream_t stream) {
  if (rows <= 0 || n_cols <= 0) return;
  // total width is the sum of the group widths: computed on the host by the caller's layout
  // (cols lives on the device), so it is passed through part_stride == total width
  const int total_width = static_cast<int>(part_stride);
  const int64_t n = rows * total_width;
  int64_t blocks = (n + 255) / 256;
  if (blocks > kGridCapSms * 8) blocks = kGridCapSms * 8;
  with_dtype(out_dtype, [&](auto out_t) {
    using OutT = typename decltype(out_t)::type;
    rowslice_reduce_kernel<OutT><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        partial, world, rows, part_stride, reinterpret_cast<OutT*>(out), out_stride, cols, n_cols,
        total_width);
  });
}

}  // namespace de
