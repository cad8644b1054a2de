// Pooled embedding lookup forward and atomic scatter-add backward for sm_90a.
//
// One persistent, descriptor-driven kernel serves every table of the rank.  A warp owns a tile
// of 32 consecutive samples of one input; inside the warp, LPR lanes cooperate on one row
// (LPR * VEC columns per pass) and 32/LPR rows are in flight side by side, with a further 4x
// unroll so that >= 4 independent 16-byte row loads per lane are outstanding (HBM3 needs ~16 KB
// in flight per SM).  Sources of ids and destinations of pooled rows are *peer-mapped* pointers:
// with world_size > 1 the kernel reads indices straight out of the requesters' staging buffers
// and stores pooled rows straight into the requesters' output tensors over NVLink (the two
// all-to-alls of the reference, dist_model_parallel.py:211 and :872, fused into the lookup).
// Tile order interleaves destination ranks (rotated by the local rank) so all NVLink egress and
// every peer's ingress stay evenly loaded instead of all GPUs bursting at peer 0.
//
// Capability parity: EmbeddingLookUpVariableHot / ...HotWide (reference
// cc/kernels/embedding_lookup_kernels.cu:175-336) + the dense tf.gather/reduce path.
#include <cstdlib>

#include "common.cuh"

namespace de {

namespace {

constexpr int kThreads = 256;
constexpr int kWarpsPerBlock = kThreads / 32;
constexpr int kTile = 32;  // samples per warp tile
constexpr int kUnroll = 4;
constexpr int kBlocksPerSM = 4;  // 64 registers / thread -> 32 resident warps per SM
// 16-bit rows read 8 columns per lane: the 4 row fragments of 8 fp32 each in flight need ~80
// registers (at 64 they spill), so these instantiations keep 3 blocks per SM
constexpr int fwd_blocks_per_sm(int vec) { return vec == 8 ? 3 : kBlocksPerSM; }

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

struct TileCoord {
  int f;        // local input
  int d;        // destination (requester) rank
  int64_t g0;   // first global sample
  int nsamp;    // samples in tile
};

__device__ __forceinline__ TileCoord decode_tile(int64_t t, int n_inputs, int n_dst,
                                                 int64_t tiles_per_dst, int64_t batch,
                                                 int64_t dst_batch, int rot, int ts = kTile) {
  TileCoord c;
  int dd = static_cast<int>(t % n_dst);
  int64_t rest = t / n_dst;
  c.f = static_cast<int>(rest % n_inputs);
  int64_t chunk = rest / n_inputs;
  c.d = (dd + rot) % n_dst;
  int64_t local0 = chunk * ts;
  c.g0 = static_cast<int64_t>(c.d) * dst_batch + local0;
  int64_t lim = min(dst_batch, batch - static_cast<int64_t>(c.d) * dst_batch);
  int64_t rem = lim - local0;
  c.nsamp = rem < ts ? static_cast<int>(rem < 0 ? 0 : rem) : ts;
  return c;
}

template <typename IdT>
struct IdReader {
  const IdT* direct;      // per-input direct pointer (global batch order) or nullptr
  const int64_t* offsets; // CSR
  const PeerPtrs* src;
  int64_t ids_off;
  int64_t src_batch;
  int hot;

  // number of ids of sample g and the pointer to its first id
  __device__ __forceinline__ const IdT* sample(int64_t g, int& n) const {
    if (offsets != nullptr) {
      int64_t a = offsets[g], b = offsets[g + 1];
      n = static_cast<int>(b - a);
      return direct + a;
    }
    n = hot;
    if (direct != nullptr) return direct + g * hot;
    int64_t s = g / src_batch;
    int64_t i = g - s * src_batch;
    return reinterpret_cast<const IdT*>(src->p[s]) + ids_off + i * hot;
  }
};

template <typename IdT>
__device__ __forceinline__ IdReader<IdT> make_reader(const InputDesc& D, const PeerPtrs& src,
                                                     int64_t src_batch) {
  IdReader<IdT> r;
  r.direct = reinterpret_cast<const IdT*>(D.ids);
  r.offsets = D.offsets;
  r.src = &src;
  r.ids_off = D.ids_off;
  r.src_batch = src_batch;
  r.hot = D.hotness;
  return r;
}

// =============================================================================== forward
template <typename IdT, typename OutT, int VEC, typename TabT>
__global__ void __launch_bounds__(kThreads, fwd_blocks_per_sm(VEC))
lookup_fwd_kernel(const InputDesc* __restrict__ descs, int n_inputs, int64_t batch,
                  int64_t src_batch, int64_t dst_batch, int64_t dst_stride,
                  const __grid_constant__ PeerPtrs src, const __grid_constant__ PeerPtrs dst,
                  int rot, const __grid_constant__ SyncArgs sync, int ts) {
  // ts = samples per warp tile (power of two <= 32): 32 for one-hot inputs; multi-hot inputs
  // get smaller tiles so that a launch still has enough warps when every sample pools tens or
  // hundreds of rows (the reference splits long reductions over blockDim.y, CU:195-226)
  sync_head(sync);  // the ids of every requester have landed in this rank's id buffer
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int n_dst = static_cast<int>((batch + dst_batch - 1) / dst_batch);
  const int64_t tiles_per_dst = (dst_batch + ts - 1) / ts;
  const int64_t total = static_cast<int64_t>(n_inputs) * n_dst * tiles_per_dst;

  for (int64_t t = warp; t < total; t += n_warps) {
    const TileCoord tc = decode_tile(t, n_inputs, n_dst, tiles_per_dst, batch, dst_batch, rot, ts);
    if (tc.nsamp <= 0) continue;
    const InputDesc D = descs[tc.f];
    const int W = D.width;
    const int nvec = (W + VEC - 1) / VEC;           // VEC==4 / 8 requires W % VEC == 0
    const int lpr = min(32, pow2_ceil(nvec));       // lanes per row
    const int rpw = 32 / lpr;                       // rows in flight per warp
    const int sub = lane / lpr, li = lane - sub * lpr;
    // fp32, bf16 or fp16 rows (one type per launch); pooling is always fp32
    const TabT* table = reinterpret_cast<const TabT*>(D.table);
    OutT* out_base = reinterpret_cast<OutT*>(dst.p[tc.d]);
    const int64_t i0 = tc.g0 - static_cast<int64_t>(tc.d) * dst_batch;
    const IdReader<IdT> rd = make_reader<IdT>(D, src, src_batch);
    const bool onehot = (D.hotness == 1) && (D.offsets == nullptr);
    const bool skip_empty = (D.flags & 1) != 0;  // row slices: only the owner of an id writes
    // one-hot: the 32 ids of the tile arrive with ONE coalesced load (lane = sample) and are
    // handed to the lane groups by shuffle - the row gathers then issue back to back instead
    // of each waiting for its own dependent id load
    long long tile_id = -1;
    if (onehot && lane < tc.nsamp) {
      int n;
      const IdT* p = rd.sample(tc.g0 + lane, n);
      tile_id = static_cast<long long>(*p) + D.id_shift;
    }

    for (int c0 = 0; c0 < nvec; c0 += lpr) {        // column pass (one pass when W <= 128)
      const int cv = c0 + li;
      const bool col_ok = cv < nvec;
      const int col = cv * VEC;
      if (onehot) {
        // 4 samples per lane group in flight
        for (int r0 = 0; r0 < tc.nsamp; r0 += rpw * kUnroll) {
          FVec<VEC> acc[kUnroll];
          bool ok[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const int r = r0 + u * rpw + sub;
            ok[u] = (r < tc.nsamp) && col_ok;
            acc[u].zero();
            const int64_t id = __shfl_sync(0xffffffffu, tile_id, r & 31);
            if (ok[u]) {
              if (static_cast<uint64_t>(id) < static_cast<uint64_t>(D.sub_rows)) {
                acc[u] = ld_tab<TabT, VEC>(table + (D.row_base + id) * W + col);
              } else if (skip_empty) {
                // row slices: another rank owns this id - unless it lies outside the whole
                // table, then the first / last shard stores the zero row (flags 2 / 4)
                const bool caught = ((D.flags & 2) && id < 0) || ((D.flags & 4) && id >= D.sub_rows);
                if (!caught) ok[u] = false;
              }
            }
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            if (ok[u]) {
              const int r = r0 + u * rpw + sub;
              st_act<OutT, VEC>(out_base + (i0 + r) * dst_stride + D.dst_col + col, acc[u]);
            }
          }
        }
      } else {
        for (int r0 = 0; r0 < tc.nsamp; r0 += rpw) {
          const int r = r0 + sub;
          if (r >= tc.nsamp || !col_ok) continue;
          int n;
          const IdT* p = rd.sample(tc.g0 + r, n);
          FVec<VEC> acc;
          acc.zero();
          int h = 0, hits = 0;
          // rows of one sample in flight (16-byte rows of 8 columns: 4, or the fragments spill)
          constexpr int kHotUnroll = VEC == 8 ? 4 : 8;
          for (; h + kHotUnroll <= n; h += kHotUnroll) {
            int64_t id[kHotUnroll];
            FVec<VEC> x[kHotUnroll];
#pragma unroll
            for (int u = 0; u < kHotUnroll; ++u)
              id[u] = static_cast<int64_t>(p[h + u]) + D.id_shift;
#pragma unroll
            for (int u = 0; u < kHotUnroll; ++u) {
              x[u].zero();
              if (static_cast<uint64_t>(id[u]) < static_cast<uint64_t>(D.sub_rows)) {
                x[u] = ld_tab<TabT, VEC>(table + (D.row_base + id[u]) * W + col);
                ++hits;
              }
            }
#pragma unroll
            for (int u = 0; u < kHotUnroll; ++u) acc.add(x[u]);
          }
          for (; h < n; ++h) {
            const int64_t id = static_cast<int64_t>(p[h]) + D.id_shift;
            if (static_cast<uint64_t>(id) < static_cast<uint64_t>(D.sub_rows)) {
              acc.add(ld_tab<TabT, VEC>(table + (D.row_base + id) * W + col));
              ++hits;
            }
          }
          if (skip_empty && hits == 0) continue;
          if (D.combiner == 1 && n > 0) acc.scale(1.0f / static_cast<float>(n));
          st_act<OutT, VEC>(out_base + (i0 + r) * dst_stride + D.dst_col + col, acc);
        }
      }
    }
  }
  sync_tail(sync);  // every pooled row of this rank is on its way: tell the requesters
}

// =============================================================================== backward
// dst_table[row] += scale * w_sample * grad_row   (vector RED, no return value)
// (the 8-column variant keeps 32 gradient floats per lane in flight: give it 128 registers,
//  at 64 it spills ~440 bytes per thread)
template <typename IdT, typename GradT, int VEC>
__global__ void __launch_bounds__(kThreads, VEC == 8 ? 2 : kBlocksPerSM)
scatter_add_bwd_kernel(const InputDesc* __restrict__ descs, int n_inputs, int64_t batch,
                       int64_t src_batch, int64_t grad_batch, int64_t grad_stride,
                       const __grid_constant__ PeerPtrs src, const __grid_constant__ PeerPtrs grad,
                       int rot, float scale, const float* __restrict__ scale_ptr,
                       const __grid_constant__ SyncArgs sync) {
  sync_head(sync);  // every requester's gradient rows have landed in the receive buffer
  if (scale_ptr != nullptr) scale *= *scale_ptr;  // device-resident lr (CUDA-graph friendly)
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int n_dst = static_cast<int>((batch + grad_batch - 1) / grad_batch);
  const int64_t tiles_per_dst = (grad_batch + kTile - 1) / kTile;
  const int64_t total = static_cast<int64_t>(n_inputs) * n_dst * tiles_per_dst;

  for (int64_t t = warp; t < total; t += n_warps) {
    const TileCoord tc = decode_tile(t, n_inputs, n_dst, tiles_per_dst, batch, grad_batch, rot);
    if (tc.nsamp <= 0) continue;
    const InputDesc D = descs[tc.f];
    const int W = D.width;
    const int nvec = (W + VEC - 1) / VEC;
    const int lpr = min(32, pow2_ceil(nvec));
    const int rpw = 32 / lpr;
    const int sub = lane / lpr, li = lane - sub * lpr;
    float* table = reinterpret_cast<float*>(const_cast<void*>(D.table));
    const GradT* grad_base = reinterpret_cast<const GradT*>(grad.p[tc.d]);
    const int64_t i0 = tc.g0 - static_cast<int64_t>(tc.d) * grad_batch;
    const IdReader<IdT> rd = make_reader<IdT>(D, src, src_batch);

    // Pull the table rows of the *next* tile of this warp into L2 so that its reductions find
    // their lines resident (an atomic that misses L2 waits for the DRAM fill at the slice).
    {
      const int64_t tn = t + n_warps;
      if (tn < total) {
        const TileCoord nc = decode_tile(tn, n_inputs, n_dst, tiles_per_dst, batch, grad_batch,
                                         rot);
        if (lane < nc.nsamp) {
          const InputDesc& N = descs[nc.f];
          const IdReader<IdT> nrd = make_reader<IdT>(N, src, src_batch);
          int nn;
          const IdT* np = nrd.sample(nc.g0 + lane, nn);
          const int lines = (N.width * 4 + 127) >> 7;
          for (int h = 0; h < min(nn, 4); ++h) {
            const int64_t id = static_cast<int64_t>(np[h]) + N.id_shift;
            if (static_cast<uint64_t>(id) < static_cast<uint64_t>(N.sub_rows)) {
              const char* row = reinterpret_cast<const char*>(N.table) +
                                (N.row_base + id) * N.width * 4;
              for (int l = 0; l < lines; ++l) prefetch_l2(row + (l << 7));
            }
          }
        }
      }
    }

    // one-hot inputs: the tile's 32 ids come with one coalesced load and are handed out by
    // shuffle, so the reductions do not wait for a dependent per-row id load
    const bool onehot = (D.hotness == 1) && (D.offsets == nullptr);
    long long tile_id = -1;
    if (onehot && lane < tc.nsamp) {
      int n0;
      const IdT* p0 = rd.sample(tc.g0 + lane, n0);
      tile_id = static_cast<long long>(*p0) + D.id_shift;
    }
    if (onehot) {
      for (int c0 = 0; c0 < nvec; c0 += lpr) {
        const int cv = c0 + li;
        const bool col_ok = cv < nvec;
        const int col = cv * VEC;
        for (int r0 = 0; r0 < tc.nsamp; r0 += rpw * kUnroll) {
          FVec<VEC> g[kUnroll];
          int64_t id[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const int r = r0 + u * rpw + sub;
            const int64_t idr = __shfl_sync(0xffffffffu, tile_id, r & 31);
            id[u] = -1;
            if (r < tc.nsamp && col_ok &&
                static_cast<uint64_t>(idr) < static_cast<uint64_t>(D.sub_rows)) {
              id[u] = idr;
              g[u] = ld_act<GradT, VEC>(grad_base + (i0 + r) * grad_stride + D.dst_col + col);
              g[u].scale(scale);
            }
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u)
            if (id[u] >= 0) red_add_f32<VEC>(table + (D.row_base + id[u]) * W + col, g[u]);
        }
      }
      continue;
    }
    for (int c0 = 0; c0 < nvec; c0 += lpr) {
      const int cv = c0 + li;
      const bool col_ok = cv < nvec;
      const int col = cv * VEC;
      for (int r0 = 0; r0 < tc.nsamp; r0 += rpw * kUnroll) {
        FVec<VEC> g[kUnroll];
        const IdT* p[kUnroll];
        int n[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int r = r0 + u * rpw + sub;
          n[u] = 0;
          p[u] = nullptr;
          if (r < tc.nsamp && col_ok) {
            p[u] = rd.sample(tc.g0 + r, n[u]);
            g[u] = ld_act<GradT, VEC>(grad_base + (i0 + r) * grad_stride + D.dst_col + col);
            float w = scale;
            if (D.combiner == 1 && n[u] > 0) w /= static_cast<float>(n[u]);
            g[u].scale(w);
          }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          for (int h = 0; h < n[u]; ++h) {
            const int64_t id = static_cast<int64_t>(p[u][h]) + D.id_shift;
            if (static_cast<uint64_t>(id) < static_cast<uint64_t>(D.sub_rows))
              red_add_f32<VEC>(table + (D.row_base + id) * W + col, g[u]);
          }
        }
      }
    }
  }
  sync_tail(sync);  // ids and gradient rows are consumed: the requesters may overwrite them
}

// ---- staged variant of the atomic SGD update -------------------------------------------------
// ncu of the kernel above (MLPerf tables, batch 65536): 60 % of the stall samples sit on the
// unpack right after the gradient-row loads - 4 rows of 8 bytes per lane in flight per warp
// (~30 KB per SM) do not cover the latency of an L2 that is busy filling lines for the
// reductions.  Here every warp streams the gradient rows of its *next* tile (32 samples x row
// bytes, up to 8 KB) into shared memory with cp.async while it reduces the current one from
// shared memory: no registers held by loads in flight, ~100 KB per SM in flight, the RED
// instructions issue back to back.  The tile's ids are fetched one tile ahead as well (one
// coalesced load, lane = sample) and its table rows are prefetched into L2.
constexpr int kStagedWarps = 7;
constexpr int kStagedThreads = kStagedWarps * 32;
constexpr int kStageBytes = 8192;  // one tile: 32 samples x <= 256 bytes of gradient row

__device__ __forceinline__ void cp_async16_g2s(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                   static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst))),
               "l"(gmem_src)
               : "memory");
}

template <typename IdT, typename GradT>
__global__ void __launch_bounds__(kStagedThreads, 2)
scatter_add_staged_kernel(const InputDesc* __restrict__ descs, int n_inputs, int64_t batch,
                          int64_t src_batch, int64_t grad_batch, int64_t grad_stride,
                          const __grid_constant__ PeerPtrs src,
                          const __grid_constant__ PeerPtrs grad, int rot, float scale,
                          const float* __restrict__ scale_ptr,
                          const __grid_constant__ SyncArgs sync) {
  extern __shared__ __align__(16) unsigned char staged_smem[];
  sync_head(sync);  // every requester's gradient rows have landed in the receive buffer
  if (scale_ptr != nullptr) scale *= *scale_ptr;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  unsigned char* stage = staged_smem + static_cast<size_t>(wib) * 2 * kStageBytes;
  const int64_t warp = static_cast<int64_t>(blockIdx.x) * kStagedWarps + wib;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kStagedWarps;
  const int n_dst = static_cast<int>((batch + grad_batch - 1) / grad_batch);
  const int64_t tiles_per_dst = (grad_batch + kTile - 1) / kTile;
  const int64_t total = static_cast<int64_t>(n_inputs) * n_dst * tiles_per_dst;

  // gradient rows (and, for one-hot inputs, the ids) of tile t -> buffer `buf`
  auto issue = [&](int64_t t, int buf, long long& ids_out) {
    const TileCoord tc = decode_tile(t, n_inputs, n_dst, tiles_per_dst, batch, grad_batch, rot);
    const InputDesc& D = descs[tc.f];
    const int row_bytes = D.width * static_cast<int>(sizeof(GradT));
    const int cpr = row_bytes >> 4;  // 16-byte chunks per row
    const int64_t i0 = tc.g0 - static_cast<int64_t>(tc.d) * grad_batch;
    const unsigned char* gbase = reinterpret_cast<const unsigned char*>(
        reinterpret_cast<const GradT*>(grad.p[tc.d]) + i0 * grad_stride + D.dst_col);
    unsigned char* dst = stage + buf * kStageBytes;
    const int n_chunks = tc.nsamp * cpr;
    for (int c = lane; c < n_chunks; c += 32) {
      const int r = c / cpr, ch = c - r * cpr;
      cp_async16_g2s(dst + r * row_bytes + (ch << 4),
                     gbase + static_cast<int64_t>(r) * grad_stride * sizeof(GradT) + (ch << 4));
    }
    ids_out = -1;
    if (D.hotness == 1 && D.offsets == nullptr && lane < tc.nsamp) {
      const IdReader<IdT> rd = make_reader<IdT>(D, src, src_batch);
      int n;
      const IdT* p = rd.sample(tc.g0 + lane, n);
      ids_out = static_cast<long long>(*p) + D.id_shift;
      // the row this sample reduces into: have it resident in L2 when the RED arrives
      if (static_cast<uint64_t>(ids_out) < static_cast<uint64_t>(D.sub_rows)) {
        const char* row = reinterpret_cast<const char*>(D.table) +
                          (D.row_base + ids_out) * D.width * 4;
        for (int l = 0; l < ((D.width * 4 + 127) >> 7); ++l) prefetch_l2(row + (l << 7));
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  long long ids_cur = -1, ids_next = -1;
  int64_t t = warp;
  int buf = 0;
  if (t < total) issue(t, 0, ids_cur);
  for (; t < total; t += n_warps, buf ^= 1) {
    const int64_t tn = t + n_warps;
    if (tn < total) issue(tn, buf ^ 1, ids_next);
    else asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncwarp();
    const TileCoord tc = decode_tile(t, n_inputs, n_dst, tiles_per_dst, batch, grad_batch, rot);
    const InputDesc D = descs[tc.f];
    const int W = D.width;
    const int nvec = W >> 2;                        // 4 columns per lane
    const int lpr = min(32, pow2_ceil(nvec));
    const int rpw = 32 / lpr;
    const int sub = lane / lpr, li = lane - sub * lpr;
    float* table = reinterpret_cast<float*>(const_cast<void*>(D.table));
    const GradT* srow = reinterpret_cast<const GradT*>(stage + buf * kStageBytes);
    const bool onehot = (D.hotness == 1) && (D.offsets == nullptr);
    const IdReader<IdT> rd = make_reader<IdT>(D, src, src_batch);
    // one-hot inputs: samples of the tile that hit the same row are summed in the warp (their
    // gradient rows are in shared memory anyway) and reduced into the table ONCE.  A table with
    // a handful of rows, or the head of a power-law id distribution, otherwise serialises
    // thousands of reductions on a few L2 lines (the rank that owns the tiny MLPerf tables
    // would take several times as long as the others).
    unsigned leaders = 0, my_peers = 0;
    if (onehot) {
      const bool valid = lane < tc.nsamp &&
                         static_cast<uint64_t>(ids_cur) < static_cast<uint64_t>(D.sub_rows);
      const long long key = valid ? ids_cur : static_cast<long long>(-2 - lane);
      my_peers = __match_any_sync(0xffffffffu, key);
      leaders = __ballot_sync(0xffffffffu, valid && lane == __ffs(my_peers) - 1);
    }
    for (int c0 = 0; c0 < nvec; c0 += lpr) {
      const int cv = c0 + li;
      const bool col_ok = cv < nvec;
      const int col = cv << 2;
      for (int r0 = 0; r0 < tc.nsamp; r0 += rpw) {
        const int r = r0 + sub;
        const bool ok = (r < tc.nsamp) && col_ok;
        if (onehot) {
          const int64_t id = __shfl_sync(0xffffffffu, ids_cur, r & 31);
          unsigned members = __shfl_sync(0xffffffffu, my_peers, r & 31);
          if (ok && ((leaders >> r) & 1u)) {
            FVec<4> g = ld_act<GradT, 4>(srow + r * W + col);
            members &= ~(1u << r);
            while (members) {  // the other samples of this tile with the same id
              const int j = __ffs(members) - 1;
              members &= members - 1;
              g.add(ld_act<GradT, 4>(srow + j * W + col));
            }
            g.scale(scale);
            red_add_f32<4>(table + (D.row_base + id) * W + col, g);
          }
        } else if (ok) {
          int n;
          const IdT* p = rd.sample(tc.g0 + r, n);
          FVec<4> g = ld_act<GradT, 4>(srow + r * W + col);
          float w = scale;
          if (D.combiner == 1 && n > 0) w /= static_cast<float>(n);
          g.scale(w);
          for (int h = 0; h < n; ++h) {
            const int64_t id = static_cast<int64_t>(p[h]) + D.id_shift;
            if (static_cast<uint64_t>(id) < static_cast<uint64_t>(D.sub_rows))
              red_add_f32<4>(table + (D.row_base + id) * W + col, g);
          }
        }
      }
    }
    ids_cur = ids_next;
    __syncwarp();  // all lanes are done with buffer `buf` before the next iteration refills it
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  sync_tail(sync);  // ids and gradient rows are consumed: the requesters may overwrite them
}

// DE_B200_EMB_BLOCKS_PER_SM=1..4 caps the resident CTAs per SM of the persistent lookup / scatter
// grids (default 4 = the launch bound): fewer CTAs leave registers and shared memory for kernels
// of other streams (the MLP GEMMs overlapped with the embedding exchange).
int blocks_per_sm_cap(int compiled) {
  static const int env = [] {
    const char* v = std::getenv("DE_B200_EMB_BLOCKS_PER_SM");
    return v != nullptr ? std::atoi(v) : 0;
  }();
  return (env >= 1 && env < compiled) ? env : compiled;
}

int grid_for(int64_t total_tiles, int sm_count, int blocks_per_sm) {
  blocks_per_sm = blocks_per_sm_cap(blocks_per_sm);
  int64_t blocks = (total_tiles + kWarpsPerBlock - 1) / kWarpsPerBlock;
  int64_t cap = static_cast<int64_t>(sm_count) * blocks_per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

int64_t count_tiles(int n_inputs, int64_t batch, int64_t dst_batch, int ts = kTile) {
  int64_t n_dst = (batch + dst_batch - 1) / dst_batch;
  int64_t tiles_per_dst = (dst_batch + ts - 1) / ts;
  return static_cast<int64_t>(n_inputs) * n_dst * tiles_per_dst;
}

}  // namespace

void launch_lookup_fwd(const InputDesc* descs, int n_inputs, int64_t batch, int64_t src_batch,
                       int64_t dst_batch, int64_t dst_stride, const PeerPtrs& src,
                       const PeerPtrs& dst, int rot, bool ids64, int act_dtype, bool vec4,
                       int sm_count, cudaStream_t stream, const SyncArgs& sync,
                       int tile_samples, int table_dtype, bool vec8) {
  if (n_inputs <= 0 || batch <= 0) {
    launch_sync_only(sync, stream);  // keep the signalling protocol in step
    return;
  }
  int ts = 1;
  while (ts * 2 <= tile_samples && ts < kTile) ts *= 2;  // power of two in [1, 32]
  // 16-bit rows: 8 columns (one 16-byte load) per lane where the widths allow it
  const int vec = !vec4 ? 1 : (vec8 && table_dtype != 0) ? 8 : 4;
  const int grid = grid_for(count_tiles(n_inputs, batch, dst_batch, ts), sm_count,
                            fwd_blocks_per_sm(vec));
  with_dtype(table_dtype, [&](auto tab) {
    using TabT = typename decltype(tab)::type;
    with_type_if<int64_t, int32_t>(ids64, [&](auto id) {
      using IdT = typename decltype(id)::type;
      with_dtype(act_dtype, [&](auto out) {
        using OutT = typename decltype(out)::type;
        auto launch = [&](auto kernel) {
          kernel<<<grid, kThreads, 0, stream>>>(descs, n_inputs, batch, src_batch, dst_batch,
                                                dst_stride, src, dst, rot, sync, ts);
        };
        if constexpr (sizeof(TabT) == 2) {
          if (vec == 8) {
            launch(lookup_fwd_kernel<IdT, OutT, 8, TabT>);
            return;
          }
        }
        if (vec == 4) launch(lookup_fwd_kernel<IdT, OutT, 4, TabT>);
        else launch(lookup_fwd_kernel<IdT, OutT, 1, TabT>);
      });
    });
  });
}

void launch_scatter_add_bwd(const InputDesc* descs, int n_inputs, int64_t batch, int64_t src_batch,
                            int64_t grad_batch, int64_t grad_stride, const PeerPtrs& src,
                            const PeerPtrs& grad, int rot, float scale, const float* scale_ptr,
                            bool ids64, int act_dtype, bool vec4, int sm_count,
                            cudaStream_t stream, bool vec8, const SyncArgs& sync, bool staged) {
  if (n_inputs <= 0 || batch <= 0) {
    launch_sync_only(sync, stream);
    return;
  }
  with_type_if<int64_t, int32_t>(ids64, [&](auto id) {
    using IdT = typename decltype(id)::type;
    with_dtype(act_dtype, [&](auto grad_t) {
      using GradT = typename decltype(grad_t)::type;
      if (staged && vec4) {
        // caller guarantees: every gradient row is a 16-byte multiple of at most 256 bytes,
        // 16-byte aligned in the source (column offsets, row stride, base pointers)
        const int64_t tiles = count_tiles(n_inputs, batch, grad_batch);
        int64_t blocks = (tiles + kStagedWarps - 1) / kStagedWarps;
        if (blocks > static_cast<int64_t>(sm_count) * 2) blocks = static_cast<int64_t>(sm_count) * 2;
        const size_t smem = static_cast<size_t>(kStagedWarps) * 2 * kStageBytes;
        cudaFuncSetAttribute(scatter_add_staged_kernel<IdT, GradT>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        scatter_add_staged_kernel<IdT, GradT>
            <<<static_cast<unsigned>(blocks), kStagedThreads, smem, stream>>>(
                descs, n_inputs, batch, src_batch, grad_batch, grad_stride, src, grad, rot, scale,
                scale_ptr, sync);
        return;
      }
      const int grid = grid_for(count_tiles(n_inputs, batch, grad_batch), sm_count, kBlocksPerSM);
      auto launch = [&](auto kernel) {
        kernel<<<grid, kThreads, 0, stream>>>(descs, n_inputs, batch, src_batch, grad_batch,
                                              grad_stride, src, grad, rot, scale, scale_ptr, sync);
      };
      if constexpr (sizeof(GradT) == 2) {
        // 16-byte gradient loads: 8 columns per lane, two rows per warp instruction
        if (vec8) {
          launch(scatter_add_bwd_kernel<IdT, GradT, 8>);
          return;
        }
      }
      if (vec4) launch(scatter_add_bwd_kernel<IdT, GradT, 4>);
      else launch(scatter_add_bwd_kernel<IdT, GradT, 1>);
    });
  });
}

}  // namespace de
