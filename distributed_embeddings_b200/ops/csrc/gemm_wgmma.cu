// Hand-written Hopper GEMM with fused epilogue for the MLP layers (sm_90a):
//
//   C[M,N] (bf16) = act( A[M,K] (bf16, K-major) x B[N,K]^T (bf16, K-major) + bias[N] )
//
// * operands are streamed by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) into a multi-stage
//   shared-memory ring guarded by full/empty mbarriers;
// * two consumer warpgroups each own 64 rows of the 128-row tile and issue asynchronous
//   wgmma.mma_async m64n128k16 (bf16 in, fp32 accumulate in registers) straight from shared-memory
//   matrix descriptors; one wgmma group stays in flight while the previous stage is released;
// * the epilogue adds the bias / applies ReLU on the register accumulators and stores bf16 pairs;
//   the dgrad epilogue (EPI 2) masks them against the ReLU output, which was copied to shared
//   memory while the main loop ran, sums the columns, and stores the tile from shared memory in
//   16-byte chunks.
// Warpgroup roles: warpgroup 0 = TMA producer (one thread), warpgroups 1..2 = MMA + epilogue.
//
// Replaces the cuBLAS GEMM + separate bias/activation ops that TF/XLA runs for the reference's
// Dense layers (examples/dlrm/main.py:123-145).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
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
// 16-byte asynchronous global -> shared copy (L2 only); src_bytes = 0 fills zeros, reads nothing
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(smem_dst)),
               "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}
// shared-memory accesses by address: the 1024-byte realignment of the dynamic window hides the
// address space from the compiler, which would otherwise emit generic loads and stores
__device__ __forceinline__ uint32_t lds_b32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_b32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 lds_b128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "r"(a)
               : "memory");
  return v;
}
__device__ __forceinline__ void red_add_f32(float* gmem, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(gmem), "f"(v) : "memory");
}
__device__ __forceinline__ void warpgroup_bar_sync(int cw) {  // the 128 threads of warpgroup 1 + cw
  asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory");
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

template <int BLOCK_N, int STAGES, int EPI = 0>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // EPI 2: each consumer warpgroup's 64 x BLOCK_N tile of the ReLU output, which the epilogue
  // overwrites with the masked result before it is stored.  Rows are padded by 16 bytes, so the
  // 8 rows x 4 words a warp touches per accumulator fragment fall into 32 different banks.
  static constexpr int kActRowBytes = BLOCK_N * 2 + 16;
  static constexpr int kActWgBytes = 64 * kActRowBytes;
  static constexpr int kActOffset = STAGES * kStageBytes;
  // EPI 2: per-warp column sums of the current tile, [consumer warp 0..7][BLOCK_N] fp32
  static constexpr int kColsumOffset = kActOffset + (EPI == 2 ? 2 * kActWgBytes : 0);
  static constexpr int kBarOffset = kColsumOffset + kMaxColsum * 4;
  static_assert(8 * BLOCK_N <= kMaxColsum, "per-warp column sums exceed their region");
  static constexpr int kNumBars = 2 * STAGES;  // full / empty per stage
  // tile index of the k block in each stage (-1: no more tiles), written by the producer
  static constexpr int kTileOffset = kBarOffset + kNumBars * 8;
  static constexpr int kTotal = kTileOffset + STAGES * 4;
};

// Dynamic tile scheduling of gemm_tn_fused_kernel: after its first tile (blockIdx.x), a CTA takes
// the next one from a device counter, so a CTA that becomes resident late (the GEMM shares the
// GPU with other streams' kernels) takes fewer tiles instead of setting the kernel's end.  Word 0
// counts handed-out tiles, word 1 the CTAs that found none left; the last of those resets both,
// so every launch (graph replays included) starts from zero.  Launches cycle through the slots,
// so kernels on different streams that run at the same time use different counters.
constexpr int kSchedSlots = 256;
__device__ unsigned int g_tile_sched[kSchedSlots][2];

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
                                              float* colsum, float (&acc)[BLOCK_N / WGMMA_N][64]) {
  using L = SmemLayout<BLOCK_N, STAGES, EPI>;
  constexpr int NB = BLOCK_N / WGMMA_N;
  const int lane = threadIdx.x & 31, warp_in_wg = (threadIdx.x >> 5) & 3;
  const bool releaser = warp_in_wg == 0 && lane == 0;
  // wgmma D fragment: register 4j + 2i + c holds row 16*warp + lane/4 + 8i, column
  // 8j + 2*(lane%4) + c of the warpgroup's 64 x 128 block
  const int row0 = m0 + cw * 64 + warp_in_wg * 16 + (lane >> 2);
  // EPI 2: the warpgroup's 64 rows of the ReLU output are copied to shared memory (16-byte
  // chunks, coalesced) while the main loop runs, so the epilogue does not wait on global memory
  uint8_t* s_act = smem + L::kActOffset + cw * L::kActWgBytes;
  const uint32_t s_act_a = smem_addr(s_act);
  const uint32_t s_part_a = smem_addr(smem + L::kColsumOffset) + cw * 4 * BLOCK_N * 4;
  constexpr int kRowChunks = BLOCK_N / 8;  // 16-byte chunks per row; N % 8 == 0: all in or out
  const int wt = threadIdx.x & 127;
  if constexpr (EPI == 2) {
    warpgroup_bar_sync(cw);  // the previous tile's stores have read the buffer
#pragma unroll 4
    for (int c = wt; c < 64 * kRowChunks; c += 128) {
      const int r = c / kRowChunks, cc = c % kRowChunks;
      const int row = m0 + cw * 64 + r, col = n0 + cc * 8;
      const bool ok = row < M && col < N;  // out of range: zeros, i.e. masked
      cp_async_16(s_act + r * L::kActRowBytes + cc * 16,
                  act + (ok ? static_cast<int64_t>(row) * ldact + col : 0), ok ? 16u : 0u);
    }
    cp_async_commit();
  }
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

  // ---- epilogue on the register accumulators
  if constexpr (EPI == 2) {
    cp_async_wait_all();
    warpgroup_bar_sync(cw);
  }
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
        if constexpr (EPI == 2) {
          // the act pair under (v0, v1) is replaced by the masked result, stored below
          const uint32_t sp = s_act_a + (row - m0 - cw * 64) * L::kActRowBytes + (col - n0) * 2;
          const uint32_t a = lds_b32(sp);  // bf16 pair, column col in the low half
          v0 = __uint_as_float(a << 16) > 0.f ? v0 : 0.f;
          v1 = __uint_as_float(a & 0xffff0000u) > 0.f ? v1 : 0.f;
          cs0 += v0;
          cs1 += v1;
          const __nv_bfloat162 r = __floats2bfloat162_rn(v0, v1);
          sts_b32(sp, *reinterpret_cast<const uint32_t*>(&r));
        } else {
          v0 += b0;
          v1 += b1;
          if (EPI == 1) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          if (row < M && col_ok)
            *reinterpret_cast<__nv_bfloat162*>(C + static_cast<int64_t>(row) * ldc + col) =
                __floats2bfloat162_rn(v0, v1);
        }
      }
      if (EPI == 2) {
        // lanes with the same lane % 4 hold the same two columns: sum the warp's 16 rows
#pragma unroll
        for (int sft = 4; sft < 32; sft <<= 1) {
          cs0 += __shfl_xor_sync(0xffffffffu, cs0, sft);
          cs1 += __shfl_xor_sync(0xffffffffu, cs1, sft);
        }
        if (lane < 4) {  // this warp's slot: plain stores, summed over the warps below
          const uint32_t sp = s_part_a + (warp_in_wg * BLOCK_N + col - n0) * 4;
          sts_b32(sp, __float_as_uint(cs0));
          sts_b32(sp + 4, __float_as_uint(cs1));
        }
      }
    }
  }
  if constexpr (EPI == 2) {  // the masked tile, in 16-byte coalesced stores
    warpgroup_bar_sync(cw);
    // column sums of the warpgroup's 64 rows: one fp32 reduction per column into colsum
    for (int c = wt; c < BLOCK_N; c += 128) {
      const uint32_t sp = s_part_a + c * 4;
      const float v = __uint_as_float(lds_b32(sp)) + __uint_as_float(lds_b32(sp + BLOCK_N * 4)) +
                      __uint_as_float(lds_b32(sp + 2 * BLOCK_N * 4)) +
                      __uint_as_float(lds_b32(sp + 3 * BLOCK_N * 4));
      if (n0 + c < N && v != 0.f) red_add_f32(colsum + n0 + c, v);
    }
#pragma unroll 4
    for (int c = wt; c < 64 * kRowChunks; c += 128) {
      const int r = c / kRowChunks, cc = c % kRowChunks;
      const int row = m0 + cw * 64 + r, col = n0 + cc * 8;
      if (row < M && col < N)
        *reinterpret_cast<uint4*>(C + static_cast<int64_t>(row) * ldc + col) =
            lds_b128(s_act_a + r * L::kActRowBytes + cc * 16);
    }
  }
}

// Persistent kernel: one CTA per SM walks the output tiles (n fastest so that concurrently
// running CTAs share A rows in L2), taking each next tile from g_tile_sched.  The producer runs up
// to STAGES k blocks ahead, across tile boundaries, so the next tile's operands stream in while
// the epilogue of this one runs; it passes each tile's index to the consumers in s_tile.
template <int BLOCK_N, int STAGES, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_fused_kernel(const __grid_constant__ CUtensorMap tma_a,
                     const __grid_constant__ CUtensorMap tma_b, const bf16* __restrict__ bias,
                     bf16* __restrict__ C, int64_t ldc, int M, int N, int K,
                     const bf16* __restrict__ act, int64_t ldact, float* __restrict__ colsum,
                     int sched_slot) {
  using L = SmemLayout<BLOCK_N, STAGES, EPI>;
  extern __shared__ uint8_t smem_raw[];
  // the swizzled tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  volatile int* s_tile = reinterpret_cast<int*>(smem + L::kTileOffset);

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
      unsigned int* sched = g_tile_sched[sched_slot];
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x;;) {
        // ask for the next tile now; the answer arrives while this one's loads are issued
        const int next = static_cast<int>(gridDim.x + atomicAdd(&sched[0], 1u));
        const bool done = tile >= num_tiles;
        const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (kb == 0) s_tile[stage] = done ? -1 : tile;
          if (done) {  // the consumers read -1 and stop
            mbar_arrive(&full_bar[stage]);
            break;
          }
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
        if (done) break;
        tile = next;
      }
      // this CTA took its last counter value: the last CTA to get here resets the counter
      __threadfence();
      if (atomicAdd(&sched[1], 1u) == gridDim.x - 1) {
        __threadfence();
        atomicExch(&sched[0], 0u);
        atomicExch(&sched[1], 0u);
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 1..2) =====================
    const int cw = wg - 1;
    float acc[BLOCK_N / WGMMA_N][64];
#pragma unroll
    for (int nb = 0; nb < BLOCK_N / WGMMA_N; ++nb)
#pragma unroll
      for (int r = 0; r < 64; ++r) acc[nb][r] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (;;) {
      mbar_wait(&full_bar[stage], phase);  // first k block of the next tile, or the end
      const int tile = s_tile[stage];
      if (tile < 0) break;
      const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
      consumer_tile<BLOCK_N, STAGES, EPI, false>(smem, full_bar, empty_bar, stage, phase, m0, n0,
                                                 num_kb, cw, bias, C, ldc, M, N, act, ldact,
                                                 colsum, acc);
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

int next_sched_slot() {
  static std::atomic<unsigned int> seq{0};
  return static_cast<int>(seq.fetch_add(1, std::memory_order_relaxed) % kSchedSlots);
}

template <int BLOCK_N, int STAGES, int EPI>
bool launch_one(const CUtensorMap& ta, const CUtensorMap& tb, const void* bias, void* C,
                int64_t ldc, int M, int N, int K, const void* act, int64_t ldact, float* colsum,
                int sm_count, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, STAGES, EPI>;
  const size_t smem = L::kTotal + 1024;
  static_assert(L::kTotal + 1024 <= 227 * 1024, "exceeds the 227 KB of shared memory per block");
  const int tiles = ((N + BLOCK_N - 1) / BLOCK_N) * ((M + BLOCK_M - 1) / BLOCK_M);
  dim3 grid(tiles < sm_count ? tiles : sm_count);
  cudaFuncSetAttribute(gemm_tn_fused_kernel<BLOCK_N, STAGES, EPI>,
                       cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  gemm_tn_fused_kernel<BLOCK_N, STAGES, EPI><<<grid, kGemmThreads, smem, stream>>>(
      ta, tb, reinterpret_cast<const bf16*>(bias), reinterpret_cast<bf16*>(C), ldc, M, N, K,
      reinterpret_cast<const bf16*>(act), ldact, colsum, next_sched_slot());
  return cudaGetLastError() == cudaSuccess;
}

// EPI 2 gives one pipeline stage to the shared-memory copy of the ReLU output (BLOCK_N = 256:
// 64 KB, 128: 32 KB)
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
  return launch_one<BLOCK_N, STAGES - 1, 2>(ta, tb, bias, C, ldc, M, N, K, act, ldact, colsum,
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
