// Hand-written Hopper GEMM with fused epilogue for the MLP layers (sm_90a):
//
//   C[M,N] (bf16) = act( A[M,K] (bf16, K-major) x B[N,K]^T (bf16, K-major) + bias[N] )
//
// * operands are streamed by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) into a multi-stage
//   shared-memory ring guarded by full/empty mbarriers;
// * two consumer warpgroups each own 64 rows of the 128-row tile and issue asynchronous
//   wgmma.mma_async m64n128k16 (bf16 in, fp32 accumulate in registers) straight from shared-memory
//   matrix descriptors; one wgmma group stays in flight while the previous stage is released;
// * the epilogue adds the bias / applies ReLU (or the ReLU-backward mask and column sums) on the
//   register accumulators and stores bf16 pairs.
// Warpgroup roles: warpgroup 0 = TMA producer (one thread), warpgroups 1..2 = MMA + epilogue.
//
// Replaces the cuBLAS GEMM + separate bias/activation ops that TF/XLA runs for the reference's
// Dense layers (examples/dlrm/main.py:123-145).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "de_b200.h"

namespace de {

namespace {

using bf16 = __nv_bfloat16;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 bytes = one swizzle row
constexpr int WGMMA_N = 128;  // one wgmma covers 64 x 128 x 16
constexpr int WGMMA_K = 16;
constexpr int kGemmThreads = 384;  // producer warpgroup + two consumer warpgroups
constexpr int kMaxColsum = 2048;   // EPI 2: N <= 2048

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {  // no PTX labels: the loop lives in C++, so any number of inlined copies is fine
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_addr(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
// wait that also acquires what other CTAs of the cluster released before arriving
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_addr(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, "
      "{%3, %4}], [%2];" ::"r"(smem_addr(smem_dst)),
      "l"(map), "r"(smem_addr(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// the same box lands at the same shared-memory offset of every CTA in cta_mask, and completes
// on the mbarrier at the same offset in each of them
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map,
                                                      uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::"
      "cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_addr(smem_dst)),
      "l"(map), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void consumer_bar_sync() {  // the 256 threads of warpgroups 1..2
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// d[64 x 128] (+)= A[smem desc, 64 x 16] * B[smem desc, 128 x 16]^T, both K-major
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b,
                                                 uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,"
      "%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
        "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]),
        "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),
        "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
        "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// Shared-memory matrix descriptor: K-major operand tile, rows of 128 bytes, SWIZZLE_128B, 8-row
// groups 1024 bytes apart (tile base 1024-byte aligned; a K step of 16 advances the start by 32 B).
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_byte_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_byte_addr & 0x3FFFF) >> 4);  // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                          // LBO (unused with swizzle) [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                  // SBO = 1024 B   [32,46)
  d |= static_cast<uint64_t>(1) << 62;                          // SWIZZLE_128B   [62,64)
  return d;
}

template <int BLOCK_N, int STAGES>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kColsumOffset = STAGES * kStageBytes;
  static constexpr int kBarOffset = kColsumOffset + kMaxColsum * 4;
  static constexpr int kNumBars = 2 * STAGES;  // full / empty per stage
  static constexpr int kTotal = kBarOffset + kNumBars * 8;
};

// Main loop + epilogue of one consumer warpgroup (cw = 0/1: rows [cw*64, cw*64+64) of the tile).
// CLUSTER: the empty barriers of both CTAs of a 2-CTA cluster are released (their producers
// multicast into this CTA's stages).
// EPI 0: C = A B^T + bias            EPI 1: C = relu(A B^T + bias)
// EPI 2 (backward of a ReLU layer's input): C = (A B^T) * (act > 0), colsum[n] += sum_m C[m, n]
//        i.e. dgrad GEMM + ReLU-backward mask + bias gradient of the layer below in one kernel.
template <int BLOCK_N, int STAGES, int EPI, bool CLUSTER>
__device__ __forceinline__ void consumer_tile(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                              int& stage, uint32_t& phase, int m0, int n0,
                                              int num_kb, int cw, const bf16* __restrict__ bias,
                                              bf16* __restrict__ C, int64_t ldc, int M, int N,
                                              const bf16* __restrict__ act, int64_t ldact,
                                              float* s_colsum, float (&acc)[BLOCK_N / WGMMA_N][64]) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  constexpr int NB = BLOCK_N / WGMMA_N;
  const int lane = threadIdx.x & 31, warp_in_wg = (threadIdx.x >> 5) & 3;
  const bool releaser = warp_in_wg == 0 && lane == 0;
  int prev_stage = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_addr(smem + stage * L::kStageBytes) + cw * 64 * 128;
    const uint32_t sb = smem_addr(smem + stage * L::kStageBytes + L::kABytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
      const uint64_t da = make_sw128_kmajor_desc(sa + k * WGMMA_K * 2);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const uint64_t db = make_sw128_kmajor_desc(sb + nb * WGMMA_N * 128 + k * WGMMA_K * 2);
        wgmma_m64n128k16(acc[nb], da, db, (kb | k) != 0 ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();  // the group of the previous k block has retired: its stage is free
    if (prev_stage >= 0 && releaser) {
      if (CLUSTER) {
        for (uint32_t r = 0; r < 2; ++r) {
          const uint32_t a = smem_addr(&empty_bar[prev_stage]);
          uint32_t remote;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(a), "r"(r));
          asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote)
                       : "memory");
        }
      } else {
        mbar_arrive(&empty_bar[prev_stage]);
      }
    }
    prev_stage = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  if (prev_stage >= 0 && releaser) {
    if (CLUSTER) {
      for (uint32_t r = 0; r < 2; ++r) {
        const uint32_t a = smem_addr(&empty_bar[prev_stage]);
        uint32_t remote;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(a), "r"(r));
        asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote)
                     : "memory");
      }
    } else {
      mbar_arrive(&empty_bar[prev_stage]);
    }
  }

  // ---- epilogue on the register accumulators. wgmma D fragment: register 4j + 2i + c holds
  // row 16*warp + lane/4 + 8i, column 8j + 2*(lane%4) + c of the warpgroup's 64 x 128 block.
  const int row0 = m0 + cw * 64 + warp_in_wg * 16 + (lane >> 2);
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
    for (int j = 0; j < WGMMA_N / 8; ++j) {
      const int col = n0 + nb * WGMMA_N + j * 8 + (lane & 3) * 2;
      const bool col_ok = col < N;
      float b0 = 0.f, b1 = 0.f;
      if (EPI != 2 && bias != nullptr && col_ok) {
        const float2 bb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + col));
        b0 = bb.x;
        b1 = bb.y;
      }
      float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = row0 + 8 * i;
        float v0 = acc[nb][4 * j + 2 * i], v1 = acc[nb][4 * j + 2 * i + 1];
        if (EPI == 2) {
          float2 af = make_float2(0.f, 0.f);
          if (row < M && col_ok)
            af = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(
                act + static_cast<int64_t>(row) * ldact + col));
          v0 = af.x > 0.f ? v0 : 0.f;
          v1 = af.y > 0.f ? v1 : 0.f;
          cs0 += v0;
          cs1 += v1;
        } else {
          v0 += b0;
          v1 += b1;
          if (EPI == 1) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
        }
        if (row < M && col_ok)
          *reinterpret_cast<__nv_bfloat162*>(C + static_cast<int64_t>(row) * ldc + col) =
              __floats2bfloat162_rn(v0, v1);
      }
      if (EPI == 2) {
        // lanes with the same lane % 4 hold the same two columns: sum the warp's 16 rows
#pragma unroll
        for (int sft = 4; sft < 32; sft <<= 1) {
          cs0 += __shfl_xor_sync(0xffffffffu, cs0, sft);
          cs1 += __shfl_xor_sync(0xffffffffu, cs1, sft);
        }
        if (lane < 4 && col_ok) {
          atomicAdd(&s_colsum[col], cs0);
          atomicAdd(&s_colsum[col + 1], cs1);
        }
      }
    }
  }
}

// Persistent kernel: one CTA per SM walks the output tiles (n fastest so that concurrently
// running CTAs share A rows in L2).  The producer runs up to STAGES k blocks ahead, across tile
// boundaries, so the next tile's operands stream in while the epilogue of this one runs.
template <int BLOCK_N, int STAGES, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_fused_kernel(const __grid_constant__ CUtensorMap tma_a,
                     const __grid_constant__ CUtensorMap tma_b, const bf16* __restrict__ bias,
                     bf16* __restrict__ C, int64_t ldc, int M, int N, int K,
                     const bf16* __restrict__ act, int64_t ldact, float* __restrict__ colsum) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  // the swizzled tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  float* s_colsum = reinterpret_cast<float*>(smem + L::kColsumOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const int tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int tiles_m = (M + BLOCK_M - 1) / BLOCK_M;
  const int num_tiles = tiles_n * tiles_m;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          tma_load_2d(sa, &tma_a, &full_bar[stage], kb * BLOCK_K, m0);
          tma_load_2d(sb, &tma_b, &full_bar[stage], kb * BLOCK_K, n0);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 1..2) =====================
    const int cw = wg - 1;
    if (EPI == 2) {
      for (int i = threadIdx.x - 128; i < kMaxColsum; i += 256) s_colsum[i] = 0.f;
      consumer_bar_sync();
    }
    float acc[BLOCK_N / WGMMA_N][64];
#pragma unroll
    for (int nb = 0; nb < BLOCK_N / WGMMA_N; ++nb)
#pragma unroll
      for (int r = 0; r < 64; ++r) acc[nb][r] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
      consumer_tile<BLOCK_N, STAGES, EPI, false>(smem, full_bar, empty_bar, stage, phase, m0, n0,
                                                 num_kb, cw, bias, C, ldc, M, N, act, ldact,
                                                 s_colsum, acc);
    }
    if (EPI == 2) {
      consumer_bar_sync();
      for (int i = threadIdx.x - 128; i < N && i < kMaxColsum; i += 256) {
        const float vsum = s_colsum[i];
        if (vsum != 0.f) atomicAdd(colsum + i, vsum);
      }
    }
  }
}

// ------------------------------------------------------------------ 2-CTA cluster variant
// Two CTAs of a cluster cooperate on a 256 x BLOCK_N tile: CTA r computes rows [r*128, r*128+128)
// from its own A rows, and the B tile is loaded once per cluster: CTA r fetches rows
// [r*BLOCK_N/2, ...) and TMA multicasts them into the same stage of both CTAs, halving the L2 ->
// SM traffic of B.  Every stage therefore fills from both producers, so a stage is free only once
// the consumers of BOTH CTAs released it: the empty barriers count four arrivals (two consumer
// warpgroups x two CTAs; the remote ones through mapa).
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// EPI 0: C = A B^T + bias, EPI 1: relu(...)
template <int BLOCK_N, int STAGES, int EPI>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kGemmThreads, 1)
gemm_tn_pair_kernel(const __grid_constant__ CUtensorMap tma_a,
                    const __grid_constant__ CUtensorMap tma_b, const bf16* __restrict__ bias,
                    bf16* __restrict__ C, int64_t ldc, int M, int N, int K) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  constexpr int kHalfB = L::kBBytes / 2;
  extern __shared__ uint8_t smem_raw[];
  // identical offsets in both CTAs: the dynamic shared memory window starts at the same address
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const uint32_t cta_rank = cluster_ctarank();
  const int pair = blockIdx.x >> 1, num_pairs = gridDim.x >> 1;
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const int tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int tiles_m = (M + 2 * BLOCK_M - 1) / (2 * BLOCK_M);
  const int num_tiles = tiles_n * tiles_m;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);   // this CTA's producer (expect_tx); bytes from both producers
      mbar_init(&empty_bar[s], 4);  // consumer warpgroups of both CTAs
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  cluster_sync_all();  // peer barriers are initialised before anything signals them

  if (wg == 0) {
    // ===================== TMA producer (both CTAs) =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = pair; tile < num_tiles; tile += num_pairs) {
        const int m0 = (tile / tiles_n) * (2 * BLOCK_M) + static_cast<int>(cta_rank) * BLOCK_M;
        const int n0 = (tile % tiles_n) * BLOCK_N + static_cast<int>(cta_rank) * (BLOCK_N / 2);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes + cta_rank * kHalfB;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          tma_load_2d(sa, &tma_a, &full_bar[stage], kb * BLOCK_K, m0);
          tma_load_2d_multicast(sb, &tma_b, &full_bar[stage], kb * BLOCK_K, n0, 0x3);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 1..2 of both CTAs) =====================
    const int cw = wg - 1;
    float acc[BLOCK_N / WGMMA_N][64];
#pragma unroll
    for (int nb = 0; nb < BLOCK_N / WGMMA_N; ++nb)
#pragma unroll
      for (int r = 0; r < 64; ++r) acc[nb][r] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = pair; tile < num_tiles; tile += num_pairs) {
      const int m0 = (tile / tiles_n) * (2 * BLOCK_M) + static_cast<int>(cta_rank) * BLOCK_M;
      const int n0 = (tile % tiles_n) * BLOCK_N;
      consumer_tile<BLOCK_N, STAGES, EPI, true>(smem, full_bar, empty_bar, stage, phase, m0, n0,
                                                num_kb, cw, bias, C, ldc, M, N, nullptr, 0,
                                                nullptr, acc);
    }
  }
  __syncthreads();
  cluster_sync_all();  // the peer still multicasts into / arrives on this CTA: nobody leaves early
}

// ------------------------------------------------------------------ host side: tensor maps
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                              const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode_fn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  return fn;
}

// 2-D bf16 row-major [rows, cols] tensor, box = [box_rows, 64 cols], 128-byte swizzle
bool make_tensor_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols,
                     int64_t row_stride_elems, int box_rows) {
  EncodeFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(row_stride_elems) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(BLOCK_K), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

template <int BLOCK_N, int STAGES, int EPI>
bool launch_one(const CUtensorMap& ta, const CUtensorMap& tb, const void* bias, void* C,
                int64_t ldc, int M, int N, int K, const void* act, int64_t ldact, float* colsum,
                int sm_count, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  const size_t smem = L::kTotal + 1024;
  static_assert(L::kTotal + 1024 <= 227 * 1024, "exceeds the 227 KB of shared memory per block");
  const int tiles = ((N + BLOCK_N - 1) / BLOCK_N) * ((M + BLOCK_M - 1) / BLOCK_M);
  dim3 grid(tiles < sm_count ? tiles : sm_count);
  cudaFuncSetAttribute(gemm_tn_fused_kernel<BLOCK_N, STAGES, EPI>,
                       cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  gemm_tn_fused_kernel<BLOCK_N, STAGES, EPI><<<grid, kGemmThreads, smem, stream>>>(
      ta, tb, reinterpret_cast<const bf16*>(bias), reinterpret_cast<bf16*>(C), ldc, M, N, K,
      reinterpret_cast<const bf16*>(act), ldact, colsum);
  return cudaGetLastError() == cudaSuccess;
}

template <int BLOCK_N, int STAGES>
bool launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const void* bias, void* C,
                int64_t ldc, int M, int N, int K, int epi, const void* act, int64_t ldact,
                float* colsum, int sm_count, cudaStream_t stream) {
  if (epi == 0)
    return launch_one<BLOCK_N, STAGES, 0>(ta, tb, bias, C, ldc, M, N, K, act, ldact, colsum,
                                          sm_count, stream);
  if (epi == 1)
    return launch_one<BLOCK_N, STAGES, 1>(ta, tb, bias, C, ldc, M, N, K, act, ldact, colsum,
                                          sm_count, stream);
  return launch_one<BLOCK_N, STAGES, 2>(ta, tb, bias, C, ldc, M, N, K, act, ldact, colsum,
                                        sm_count, stream);
}

}  // namespace

// C = epilogue(A B^T). A [M,K] (lda), B [N,K] (ldb), C [M,N] (ldc): bf16, 16-byte aligned rows.
// epi 0: + bias; 1: relu(+ bias); 2: * (act > 0) and colsum[n] += column sums (N <= 2048).
bool launch_gemm_tn_fused(const void* A, int64_t lda, const void* B, int64_t ldb, const void* bias,
                          void* C, int64_t ldc, int M, int N, int K, int epi, const void* act,
                          int64_t ldact, float* colsum, int block_n, int sm_count,
                          cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return true;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return false;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) |
       reinterpret_cast<uintptr_t>(C)) & 15)
    return false;
  if (epi == 2 && (act == nullptr || colsum == nullptr || N > kMaxColsum || (ldact % 8) ||
                   (reinterpret_cast<uintptr_t>(act) & 15)))
    return false;
  const int bn = (block_n == 128 || block_n == 256) ? block_n : (N >= 256 ? 256 : 128);
  alignas(64) CUtensorMap ta, tb;
  if (!make_tensor_map(&ta, A, M, K, lda, BLOCK_M)) return false;
  if (!make_tensor_map(&tb, B, N, K, ldb, bn)) return false;
  if (bn == 256)
    return launch_cfg<256, 4>(ta, tb, bias, C, ldc, M, N, K, epi, act, ldact, colsum, sm_count,
                              stream);
  return launch_cfg<128, 6>(ta, tb, bias, C, ldc, M, N, K, epi, act, ldact, colsum, sm_count,
                            stream);
}

namespace {
template <int EPI>
bool launch_pair(const CUtensorMap& ta, const CUtensorMap& tb, const void* bias, void* C,
                 int64_t ldc, int M, int N, int K, int sm_count, cudaStream_t stream) {
  constexpr int BN = 256, ST = 4;
  using L = SmemLayout<BN, ST>;
  const size_t smem = L::kTotal + 1024;
  const int tiles = ((N + BN - 1) / BN) * ((M + 2 * BLOCK_M - 1) / (2 * BLOCK_M));
  int pairs = sm_count / 2;
  if (tiles < pairs) pairs = tiles;
  if (pairs < 1) return false;
  cudaFuncSetAttribute(gemm_tn_pair_kernel<BN, ST, EPI>,
                       cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  gemm_tn_pair_kernel<BN, ST, EPI><<<dim3(2 * pairs), kGemmThreads, smem, stream>>>(
      ta, tb, reinterpret_cast<const bf16*>(bias), reinterpret_cast<bf16*>(C), ldc, M, N, K);
  return cudaGetLastError() == cudaSuccess;
}
}  // namespace

// 2-CTA cluster kernel (256 x 256 tile per cluster, B multicast); epi 0 / 1 only.
bool launch_gemm_tn_pair(const void* A, int64_t lda, const void* B, int64_t ldb, const void* bias,
                         void* C, int64_t ldc, int M, int N, int K, bool relu, int sm_count,
                         cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return true;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return false;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) |
       reinterpret_cast<uintptr_t>(C)) & 15)
    return false;
  alignas(64) CUtensorMap ta, tb;
  if (!make_tensor_map(&ta, A, M, K, lda, BLOCK_M)) return false;
  if (!make_tensor_map(&tb, B, N, K, ldb, 128)) return false;  // each CTA fetches half the tile
  return relu ? launch_pair<1>(ta, tb, bias, C, ldc, M, N, K, sm_count, stream)
              : launch_pair<0>(ta, tb, bias, C, ldc, M, N, K, sm_count, stream);
}

bool launch_gemm_tn_bias_act(const void* A, int64_t lda, const void* B, int64_t ldb,
                             const void* bias, void* C, int64_t ldc, int M, int N, int K,
                             bool relu, int block_n, int sm_count, cudaStream_t stream) {
  // block_n == 512 selects the 2-CTA cluster kernel
  if (block_n == 512)
    return launch_gemm_tn_pair(A, lda, B, ldb, bias, C, ldc, M, N, K, relu, sm_count, stream);
  return launch_gemm_tn_fused(A, lda, B, ldb, bias, C, ldc, M, N, K, relu ? 1 : 0, nullptr, 0,
                              nullptr, block_n, sm_count, stream);
}

}  // namespace de
