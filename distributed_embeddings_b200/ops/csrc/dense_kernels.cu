// Dense-side kernels of the DLRM step for sm_90a (everything around the MLP GEMMs):
//   * dot interaction forward / backward: per sample Gram matrix F F^T of the (n_emb + 1) x D
//     feature matrix on tensor cores (mma.sync m16n8k16 bf16, one warp per sample).  The op is
//     HBM bound (7 KB in, 1 KB out per sample), the MMA only has to keep up with the loads.  The
//     backward writes the embedding gradient straight into the (symmetric) gradient buffer of
//     the embedding engine, so no extra pack / copy precedes the backward all-to-all.
//   * fused ReLU-backward + bias gradient, fused final layer + BCE loss + their backward,
//     fused SGD update of the fp32 master weights + bf16 shadow copy, input cast/pad.
//
// Capability parity: dot_interact (reference examples/dlrm/utils.py:92-113) and the TF / XLA
// elementwise + optimizer kernels the reference borrows.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>

#include "common.cuh"
#include "de_b200.h"

namespace de {

namespace {

using bf16 = __nv_bfloat16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int kMaxFeat = 32;     // rows of F incl. the bottom-MLP vector, padded to 32
constexpr int kWarps = 4;        // samples in flight per block
// Samples in flight per block of interact_bwd_apply_kernel (one 139.8 KB block per SM at n_emb
// 26).  At the step's shapes with 10 applied tables it beats 3 blocks x 4 warps and 5 x 2 per SM
// (DESIGN §8); the backward without the update is fastest at kWarps.
constexpr int kApplyWarps = 8;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// Stage F = [bottom ; emb_0 .. emb_{n-1}] (each D bf16) of one sample into rows 0..n_emb of sF with
// cp.async (LDGSTS): every 16-byte chunk of the sample is in flight before the first wait.
// Rows past n_emb are not touched: v1 zeroes them once, the forward reads a zero row instead.
template <int D>
__device__ __forceinline__ void stage_features(bf16* sF, int LD, const bf16* bottom,
                                               const bf16* emb, int n_emb, int lane) {
  constexpr int kChunks = D / 8;  // 16-byte chunks per row
  const int total = (n_emb + 1) * kChunks;
#pragma unroll 4
  for (int c = lane; c < total; c += 32) {
    const int row = c / kChunks, ch = c - row * kChunks;
    const bf16* src = row == 0 ? bottom + ch * 8 : emb + (row - 1) * D + ch * 8;
    cp_async16(sF + row * LD + ch * 8, src);
  }
  cp_async_wait_all();
}

template <int D>
__device__ __forceinline__ void zero_pad_rows(bf16* sF, int LD, int n_emb, int lane) {
  constexpr int kChunks = D / 8;
  for (int c = (n_emb + 1) * kChunks + lane; c < kMaxFeat * kChunks; c += 32) {
    const int row = c / kChunks, ch = c - row * kChunks;
    *reinterpret_cast<uint4*>(sF + row * LD + ch * 8) = make_uint4(0, 0, 0, 0);
  }
}

// Shared memory of the forward: the triangle table (C offset i * 33 + j of every z column
// idx = i (i - 1) / 2 + j < n_inter), the zero row, then per warp the nf staged rows of F.  After
// the MMAs, C = F F^T ([32][33] fp32) overwrites F from row 1 on; row 0, the bottom vector that
// z also carries, stays.
constexpr int kFwdTriBytes = kMaxFeat * (kMaxFeat - 1) / 2 * 2;  // 496 uint16, 16-byte multiple
__host__ __device__ constexpr int fwd_head_bytes(int d) { return kFwdTriBytes + (d + 8) * 2; }
__host__ __device__ constexpr int fwd_warp_bytes(int d, int n_emb) {
  return ((n_emb + 1) * (d + 8) * 2 > (d + 8) * 2 + kMaxFeat * 33 * 4)
             ? (n_emb + 1) * (d + 8) * 2
             : (d + 8) * 2 + kMaxFeat * 33 * 4;
}

// z[s] = [ tril(F F^T, -1) (row major) | bottom | 0 pad ]
template <int D>
__global__ void __launch_bounds__(kWarps * 32)
interact_fwd_kernel(const bf16* __restrict__ bottom, int64_t bottom_stride,
                    const bf16* __restrict__ emb, int64_t emb_stride, int n_emb,
                    bf16* __restrict__ z, int64_t z_stride, int z_width, int64_t batch,
                    const __grid_constant__ SyncArgs sync) {
  sync_head(sync);  // every owner's pooled rows have landed in this rank's embedding output
  constexpr int LD = D + 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nf = n_emb + 1;
  const int n_inter = nf * (nf - 1) / 2;
  uint16_t* sTri = reinterpret_cast<uint16_t*>(smem_raw);
  bf16* sZero = reinterpret_cast<bf16*>(smem_raw + kFwdTriBytes);
  bf16* sF = reinterpret_cast<bf16*>(smem_raw + fwd_head_bytes(D) +
                                     warp * fwd_warp_bytes(D, n_emb));
  float* sC = reinterpret_cast<float*>(sF + LD);  // C after the MMAs, behind row 0
  for (int idx = threadIdx.x; idx < n_inter; idx += blockDim.x) {
    int i = static_cast<int>((1.0f + sqrtf(1.0f + 8.0f * idx)) * 0.5f);
    while (i * (i - 1) / 2 > idx) --i;
    while ((i + 1) * i / 2 <= idx) ++i;
    sTri[idx] = static_cast<uint16_t>(i * 33 + idx - i * (i - 1) / 2);
  }
  for (int c = threadIdx.x; c < LD; c += blockDim.x) sZero[c] = __float2bfloat16_rn(0.f);
  __syncthreads();
  // operand rows >= nf read the zero row
  const int arow = lane & 15, brow = (lane & 7) + ((lane >> 4) << 3);
  const bf16* pa0 = arow < nf ? sF + arow * LD : sZero;
  const bf16* pa1 = 16 + arow < nf ? sF + (16 + arow) * LD : sZero;
  const bf16* pb0 = brow < nf ? sF + brow * LD : sZero;
  const bf16* pb1 = 16 + brow < nf ? sF + (16 + brow) * LD : sZero;
  // element e of a z row: triangle, bottom (row 0 of F), zero pad
  auto z_elem = [&](int e) -> bf16 {
    if (e < n_inter) return __float2bfloat16_rn(sC[sTri[e]]);
    if (e < n_inter + D) return sF[e - n_inter];
    return __float2bfloat16_rn(0.f);
  };
  const bool vec = ((reinterpret_cast<uintptr_t>(z) & 15) | (z_stride & 7)) == 0;
  const int n_vec = vec ? z_width >> 3 : 0;  // 16-byte chunks per row; the rest is stored scalar

  for (int64_t s = static_cast<int64_t>(blockIdx.x) * kWarps + warp; s < batch;
       s += static_cast<int64_t>(gridDim.x) * kWarps) {
    stage_features<D>(sF, LD, bottom + s * bottom_stride, emb + s * emb_stride, n_emb, lane);
    __syncwarp();
    // lower triangle tiles: m-tile 0 x n-tiles {0,1}; m-tile 1 x n-tiles {0..3}
    float acc0[2][4] = {}, acc1[4][4] = {};
#pragma unroll
    for (int k = 0; k < D; k += 16) {
      uint32_t a0[4], a1[4], b01[4], b23[4];
      const int acol = k + ((lane >> 4) << 3);
      ldmatrix_x4(a0, smem_u32(pa0 + acol));
      ldmatrix_x4(a1, smem_u32(pa1 + acol));
      const int bcol = k + (((lane >> 3) & 1) << 3);
      ldmatrix_x4(b01, smem_u32(pb0 + bcol));  // n-tiles 0,1 (rows 0..15)
      ldmatrix_x4(b23, smem_u32(pb1 + bcol));  // n-tiles 2,3 (rows 16..31)
      mma_bf16(acc0[0], a0, b01[0], b01[1]);
      mma_bf16(acc0[1], a0, b01[2], b01[3]);
      mma_bf16(acc1[0], a1, b01[0], b01[1]);
      mma_bf16(acc1[1], a1, b01[2], b01[3]);
      mma_bf16(acc1[2], a1, b23[0], b23[1]);
      mma_bf16(acc1[3], a1, b23[2], b23[3]);
    }
    __syncwarp();
    const int cr = lane >> 2, cc = (lane & 3) << 1;
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      sC[cr * 33 + nt * 8 + cc] = acc0[nt][0];
      sC[cr * 33 + nt * 8 + cc + 1] = acc0[nt][1];
      sC[(cr + 8) * 33 + nt * 8 + cc] = acc0[nt][2];
      sC[(cr + 8) * 33 + nt * 8 + cc + 1] = acc0[nt][3];
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      sC[(16 + cr) * 33 + nt * 8 + cc] = acc1[nt][0];
      sC[(16 + cr) * 33 + nt * 8 + cc + 1] = acc1[nt][1];
      sC[(24 + cr) * 33 + nt * 8 + cc] = acc1[nt][2];
      sC[(24 + cr) * 33 + nt * 8 + cc + 1] = acc1[nt][3];
    }
    __syncwarp();
    bf16* zp = z + s * z_stride;
    for (int c = lane; c < n_vec; c += 32) {
      uint32_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        w[k] = static_cast<uint32_t>(__bfloat16_as_ushort(z_elem(c * 8 + 2 * k))) |
               (static_cast<uint32_t>(__bfloat16_as_ushort(z_elem(c * 8 + 2 * k + 1))) << 16);
      *reinterpret_cast<uint4*>(zp + c * 8) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    for (int e = n_vec * 8 + lane; e < z_width; e += 32) zp[e] = z_elem(e);
    __syncwarp();
  }
  sync_tail(sync);
}

// dF = G F with G symmetric (G_ij = dz[idx(i,j)], zero diagonal); row 0 (+ the direct copy path)
// is the gradient of the bottom-MLP output, rows 1.. go to the embedding gradient buffer.
template <int D>
__global__ void __launch_bounds__(kWarps * 32)
interact_bwd_kernel(const bf16* __restrict__ bottom, int64_t bottom_stride,
                    const bf16* __restrict__ emb, int64_t emb_stride, int n_emb,
                    const bf16* __restrict__ dz, int64_t dz_stride, bf16* __restrict__ dbottom,
                    int64_t dbottom_stride, bf16* __restrict__ demb, int64_t demb_stride,
                    float emb_grad_scale, int64_t batch) {
  constexpr int LD = D + 8;
  constexpr int LDG = 40;  // G row stride (32 + 8 pad)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  bf16* sF = reinterpret_cast<bf16*>(smem_raw) + warp * (kMaxFeat * LD + kMaxFeat * LDG);
  bf16* sG = sF + kMaxFeat * LD;
  const int nf = n_emb + 1;
  const int n_inter = nf * (nf - 1) / 2;
  zero_pad_rows<D>(sF, LD, n_emb, lane);

  for (int64_t s = static_cast<int64_t>(blockIdx.x) * kWarps + warp; s < batch;
       s += static_cast<int64_t>(gridDim.x) * kWarps) {
    stage_features<D>(sF, LD, bottom + s * bottom_stride, emb + s * emb_stride, n_emb, lane);
    const bf16* dzp = dz + s * dz_stride;
    for (int c = lane; c < kMaxFeat * LDG / 8; c += 32)
      reinterpret_cast<uint4*>(sG)[c] = make_uint4(0, 0, 0, 0);
    __syncwarp();
    for (int idx = lane; idx < n_inter; idx += 32) {
      int i = static_cast<int>((1.0f + sqrtf(1.0f + 8.0f * idx)) * 0.5f);
      while (i * (i - 1) / 2 > idx) --i;
      while ((i + 1) * i / 2 <= idx) ++i;
      const int j = idx - i * (i - 1) / 2;
      const bf16 v = dzp[idx];
      sG[i * LDG + j] = v;
      sG[j * LDG + i] = v;
    }
    __syncwarp();
    // A = G (32x32): 2 m-tiles x 2 k-steps, loaded once
    uint32_t ga[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
        ldmatrix_x4(ga[mt][ks],
                    smem_u32(sG + (mt * 16 + (lane & 15)) * LDG + ks * 16 + ((lane >> 4) << 3)));
    const int cr = lane >> 2, cc = (lane & 3) << 1;
    bf16* dbp = dbottom + s * dbottom_stride;
    bf16* dep = demb + s * demb_stride;
#pragma unroll 1
    for (int n0 = 0; n0 < D; n0 += 32) {  // 4 n-tiles (32 columns) per pass
      float acc[2][4][4] = {};
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t b01[4], b23[4];
        // B = F as K x N row major -> transposed loads
        const int krow = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
        const int ncol = n0 + ((lane >> 4) << 3);
        ldmatrix_x4_trans(b01, smem_u32(sF + krow * LD + ncol));
        ldmatrix_x4_trans(b23, smem_u32(sF + krow * LD + ncol + 16));
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_bf16(acc[mt][0], ga[mt][ks], b01[0], b01[1]);
          mma_bf16(acc[mt][1], ga[mt][ks], b01[2], b01[3]);
          mma_bf16(acc[mt][2], ga[mt][ks], b23[0], b23[1]);
          mma_bf16(acc[mt][3], ga[mt][ks], b23[2], b23[3]);
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mt * 16 + cr + half * 8;
            const int col = n0 + nt * 8 + cc;
            float v0 = acc[mt][nt][half * 2], v1 = acc[mt][nt][half * 2 + 1];
            if (row == 0) {
              // + gradient of the direct concat path z[n_inter + col]
              v0 += __bfloat162float(dzp[n_inter + col]);
              v1 += __bfloat162float(dzp[n_inter + col + 1]);
              *reinterpret_cast<__nv_bfloat162*>(dbp + col) = __floats2bfloat162_rn(v0, v1);
            } else if (row <= n_emb) {
              *reinterpret_cast<__nv_bfloat162*>(dep + (row - 1) * D + col) =
                  __floats2bfloat162_rn(v0 * emb_grad_scale, v1 * emb_grad_scale);
            }
          }
        }
      }
    }
    __syncwarp();
  }
}

// ---- v2 of the interaction backward (the default).  v1 stalls mostly on long_scoreboard with few
// warps active - a warp loads a sample, waits, computes, stores, and only then touches the next
// sample.  v2 keeps the *next* sample's features and dz row in flight (cp.async into a second
// buffer) while the current one is multiplied and stored, and reads dz from shared memory
// (16-byte chunks) instead of 351 scalar global loads.  Only the nf = n_emb + 1 rows of F are
// staged; the MMA operand rows >= nf read one shared zero row, and the G fragments are gathered
// straight from the staged dz through a per-block offset table, so a warp holds ~16.4 KB at
// n_emb 26, dim 128: three 4-warp blocks of v2 fit on an SM.
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait_group() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

constexpr int kDzMax = 512;        // staged dz elements per sample (n_inter + D <= 512)
constexpr int kDzBuf = kDzMax + 8;  // + one zero chunk: element kDzMax reads as 0 (G's sentinel)

// Shared memory of the v2 backward, in this order: the G offset table (4 x 32 uint4: 8 dz
// offsets per lane per entry), the zero row, the applied / routed feature lists, the per-warp
// double buffers (2 x [nf][D + 8] F rows, 2 x kDzBuf dz), the chunk routing table.
constexpr int kBwdGOffBytes = 4 * 32 * 16;
constexpr int kBwdListBytes = 64;
__host__ __device__ constexpr int bwd_zero_row_bytes(int d) { return (d + 8) * 2; }
__host__ __device__ constexpr int bwd_head_bytes(int d) {
  return kBwdGOffBytes + bwd_zero_row_bytes(d) + kBwdListBytes;
}
__host__ __device__ constexpr int bwd_warp_bytes(int d, int n_emb) {
  return (2 * (n_emb + 1) * (d + 8) + 2 * kDzBuf) * 2;
}

template <int D>
__device__ __forceinline__ void issue_sample(bf16* sF, int LD, bf16* sDz, const bf16* bottom,
                                             const bf16* emb, const bf16* dz, int n_emb,
                                             int dz_chunks, int lane) {
  constexpr int kChunks = D / 8;
  const int total = (n_emb + 1) * kChunks;
#pragma unroll 4
  for (int c = lane; c < total; c += 32) {
    const int row = c / kChunks, ch = c - row * kChunks;
    const bf16* src = row == 0 ? bottom + ch * 8 : emb + (row - 1) * D + ch * 8;
    cp_async16(sF + row * LD + ch * 8, src);
  }
  for (int c = lane; c < dz_chunks; c += 32) cp_async16(sDz + c * 8, dz + c * 8);
}

// Per-block table of where every 16-byte chunk of a sample's embedding-gradient row goes:
// address of the chunk for local sample 0 and the byte stride between samples.  Built once per
// block from the route pieces (or from the single local buffer).
struct ChunkDst {
  unsigned long long base;
  long long stride;
};

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// APPLY: rows of F flagged in `apply.mask` are reduced into their table rows (SGD) instead of
// being stored through the routes; the routed rows are unchanged.
template <int D, int W, bool APPLY>
__device__ __forceinline__ void
interact_bwd_v2_body(const bf16* __restrict__ bottom, int64_t bottom_stride,
                     const bf16* __restrict__ emb, int64_t emb_stride, int n_emb,
                     const bf16* __restrict__ dz, int64_t dz_stride, bf16* __restrict__ dbottom,
                     int64_t dbottom_stride, bf16* __restrict__ demb, int64_t demb_stride,
                     float emb_grad_scale, int64_t batch, const GradRoute* __restrict__ routes,
                     int n_routes, const SyncArgs& sync, uint32_t* __restrict__ done_counters,
                     int chunk_rows, const InteractApply& apply) {
  constexpr int LD = D + 8;
  constexpr int kRowChunks = D / 8;  // 16-byte chunks per feature row
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nf = n_emb + 1;
  const int n_inter = nf * (nf - 1) / 2;
  const int dz_chunks = (n_inter + D + 7) >> 3;
  uint4* sGOff = reinterpret_cast<uint4*>(smem_raw);  // [4][32]
  bf16* sZero = reinterpret_cast<bf16*>(smem_raw + kBwdGOffBytes);
  uint8_t* sRouted = smem_raw + kBwdGOffBytes + bwd_zero_row_bytes(D);  // [32]
  uint8_t* sApplied = sRouted + 32;                                      // [32]
  const int warp_elems = bwd_warp_bytes(D, n_emb) / 2;
  bf16* base = reinterpret_cast<bf16*>(smem_raw + bwd_head_bytes(D)) + warp * warp_elems;
  bf16* sDz0 = base + 2 * nf * LD;
  ChunkDst* sDst = reinterpret_cast<ChunkDst*>(smem_raw + bwd_head_bytes(D) +
                                               W * bwd_warp_bytes(D, n_emb));
  // chunk routing table (all chunks are covered: the host checks that the pieces tile the row)
  if (routes == nullptr) {
    for (int c = threadIdx.x; c < n_emb * kRowChunks; c += blockDim.x) {
      sDst[c].base = reinterpret_cast<unsigned long long>(demb + c * 8);
      sDst[c].stride = demb_stride * 2;
    }
  } else {
    for (int r = 0; r < n_routes; ++r) {
      const GradRoute R = routes[r];
      const int c0 = R.src_col >> 3, nc = R.width >> 3;
      for (int c = threadIdx.x; c < nc; c += blockDim.x) {
        sDst[c0 + c].base =
            reinterpret_cast<unsigned long long>(reinterpret_cast<bf16*>(R.dst) + R.dst_col + c * 8);
        sDst[c0 + c].stride = R.dst_stride * 2;
      }
    }
  }
  // G offset table: A fragment register r (m-tile mt, k-step ks, 8x8 matrix q) of lane l holds
  // G[i][j], G[i][j + 1] with i = 16 mt + 8 (q & 1) + l / 4, j = 16 ks + 8 (q >> 1) + 2 (l % 4),
  // the layout ldmatrix_x4 produces.  G_ij = dz[idx(max, min)]; diagonal and pad entries point at
  // the zero element kDzMax of the dz buffer.
  for (int e = threadIdx.x; e < 4 * 32 * 8; e += blockDim.x) {
    const int l = e & 31, slot = e >> 5;  // slot = 2 * r + h, r = (mt * 2 + ks) * 4 + q
    const int h = slot & 1, r = slot >> 1, q = r & 3, ks = (r >> 2) & 1, mt = r >> 3;
    const int i = mt * 16 + (q & 1) * 8 + (l >> 2);
    const int j = ks * 16 + (q >> 1) * 8 + 2 * (l & 3) + h;
    const int hi = i > j ? i : j, lo = i > j ? j : i;
    const int off = (i == j || hi >= nf) ? kDzMax : hi * (hi - 1) / 2 + lo;
    reinterpret_cast<uint16_t*>(sGOff)[((slot >> 3) * 32 + l) * 8 + (slot & 7)] =
        static_cast<uint16_t>(off);
  }
  for (int c = threadIdx.x; c < LD; c += blockDim.x) sZero[c] = __float2bfloat16_rn(0.f);
  if (threadIdx.x == 0) {
    int na = 0, nr = 0;
    for (int f = 0; f < n_emb; ++f) {
      if (APPLY && ((apply.mask >> f) & 1u)) sApplied[na++] = static_cast<uint8_t>(f);
      else sRouted[nr++] = static_cast<uint8_t>(f);
    }
  }
  if (lane < 2)  // the zero chunk behind each of the warp's two dz buffers
    *reinterpret_cast<uint4*>(sDz0 + lane * kDzBuf + kDzMax) = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int n_applied = APPLY ? __popc(apply.mask) : 0;
  const int n_routed_chunks = (n_emb - n_applied) * kRowChunks;

  // APPLY: lane f holds the fp32 table row that feature f of the current / next sample reduces
  // into (0: not applied or id out of range)
  float apply_scale = 0.f;
  unsigned long long row_cur = 0, row_next = 0;
  if constexpr (APPLY) {
    apply_scale = apply.scale;
    if (apply.scale_ptr != nullptr) apply_scale *= *apply.scale_ptr;
  }
  auto load_row = [&](int64_t smp) -> unsigned long long {
    if (lane < n_emb && ((apply.mask >> lane) & 1u)) {
      const long long raw = apply.ids64 ? static_cast<const int64_t*>(apply.ids[lane])[smp]
                                        : static_cast<const int32_t*>(apply.ids[lane])[smp];
      const long long id = raw + apply.id_shift[lane];
      if (static_cast<unsigned long long>(id) < static_cast<unsigned long long>(apply.sub_rows[lane]))
        return reinterpret_cast<unsigned long long>(apply.table[lane] +
                                                    (apply.row_base[lane] + id) * D);
    }
    return 0;
  };
  // the row this lane's feature reduces into: have it resident in L2 when the REDs arrive
  auto prefetch_row = [&](unsigned long long row) {
    if (row != 0) {
#pragma unroll
      for (int l = 0; l < D * 4 / 128; ++l)
        prefetch_l2(reinterpret_cast<const char*>(row) + (l << 7));
    }
  };

  const int64_t stride = static_cast<int64_t>(gridDim.x) * W;
  int64_t s = static_cast<int64_t>(blockIdx.x) * W + warp;
  int cur = 0;
  if (s < batch) {
    issue_sample<D>(base, LD, sDz0, bottom + s * bottom_stride, emb + s * emb_stride,
                    dz + s * dz_stride, n_emb, dz_chunks, lane);
    if constexpr (APPLY) {
      row_cur = load_row(s);
      prefetch_row(row_cur);
    }
  }
  cp_async_commit();
  for (; s < batch; s += stride, cur ^= 1) {
    const int64_t nxt = s + stride;
    if (nxt < batch) {
      issue_sample<D>(base + (cur ^ 1) * (nf * LD), LD, sDz0 + (cur ^ 1) * kDzBuf,
                      bottom + nxt * bottom_stride, emb + nxt * emb_stride, dz + nxt * dz_stride,
                      n_emb, dz_chunks, lane);
      if constexpr (APPLY) row_next = load_row(nxt);  // consumed after this sample's MMAs
    } else if constexpr (APPLY) {
      row_next = 0;
    }
    cp_async_commit();        // possibly empty: keeps the group arithmetic uniform
    cp_async_wait_group<1>();  // everything but the prefetch just issued has landed
    __syncwarp();
    bf16* sF = base + cur * (nf * LD);
    const bf16* sDz = sDz0 + cur * kDzBuf;
    // A = G (32x32): 2 m-tiles x 2 k-steps, gathered from dz
    uint32_t ga[2][2][4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const uint4 o = sGOff[g * 32 + lane];
      const uint32_t w[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int r = g * 4 + k;
        const uint32_t lo = reinterpret_cast<const uint16_t*>(sDz)[w[k] & 0xffffu];
        const uint32_t hi = reinterpret_cast<const uint16_t*>(sDz)[w[k] >> 16];
        ga[r >> 3][(r >> 2) & 1][r & 3] = lo | (hi << 16);
      }
    }
    const int cr = lane >> 2, cc = (lane & 3) << 1;
    // B = F as K x N row major -> transposed loads; K rows >= nf read the zero row
    const bf16* brow[2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int krow = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
      brow[ks] = krow < nf ? sF + krow * LD : sZero;
    }
#pragma unroll 1
    for (int n0 = 0; n0 < D; n0 += 32) {
      float acc[2][4][4] = {};
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t b01[4], b23[4];
        const int ncol = n0 + ((lane >> 4) << 3);
        ldmatrix_x4_trans(b01, smem_u32(brow[ks] + ncol));
        ldmatrix_x4_trans(b23, smem_u32(brow[ks] + ncol + 16));
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_bf16(acc[mt][0], ga[mt][ks], b01[0], b01[1]);
          mma_bf16(acc[mt][1], ga[mt][ks], b01[2], b01[3]);
          mma_bf16(acc[mt][2], ga[mt][ks], b23[0], b23[1]);
          mma_bf16(acc[mt][3], ga[mt][ks], b23[2], b23[3]);
        }
      }
      // dF overwrites F in place: columns [n0, n0 + 32) are read by this pass only (the ldmatrix
      // loads above are warp collective, so every lane has its operands before any lane stores)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mt * 16 + cr + half * 8;
            const int col = n0 + nt * 8 + cc;
            float v0 = acc[mt][nt][half * 2], v1 = acc[mt][nt][half * 2 + 1];
            if (row == 0) {
              v0 += __bfloat162float(sDz[n_inter + col]);
              v1 += __bfloat162float(sDz[n_inter + col + 1]);
            } else {
              v0 *= emb_grad_scale;
              v1 *= emb_grad_scale;
            }
            if (row <= n_emb)
              *reinterpret_cast<__nv_bfloat162*>(sF + row * LD + col) =
                  __floats2bfloat162_rn(v0, v1);
          }
        }
      }
    }
    __syncwarp();
    if constexpr (APPLY) prefetch_row(row_next);
    // coalesced 16-byte copy-out: row 0 -> bottom-MLP gradient, routed rows -> the chunk's owner
    // (local buffer, or a peer's receive buffer over NVLink: 128-256 contiguous bytes per piece)
    if (lane < kRowChunks)
      *reinterpret_cast<uint4*>(dbottom + s * dbottom_stride + lane * 8) =
          *reinterpret_cast<const uint4*>(sF + lane * 8);
    for (int c = lane; c < n_routed_chunks; c += 32) {
      const int f = sRouted[c / kRowChunks], ch = c % kRowChunks;
      const ChunkDst d = sDst[f * kRowChunks + ch];
      *reinterpret_cast<uint4*>(d.base + static_cast<unsigned long long>(s * d.stride)) =
          *reinterpret_cast<const uint4*>(sF + (f + 1) * LD + ch * 8);
    }
    if constexpr (APPLY) {
      // applied rows, one warp instruction per row: lane l reduces floats [4l, 4l + 4) of the bf16
      // gradient the routed store would write, widened and scaled like the scatter's
      // (bf16 -> fp32, * scale), so every 32-byte sector of the table row gets one request
      static_assert(D == 128, "one red.v4 per lane covers a 128-wide row");
      for (int k = 0; k < n_applied; ++k) {
        const int f = sApplied[k];
        const unsigned long long row = __shfl_sync(0xffffffffu, row_cur, f);
        if (row == 0) continue;
        const uint2 v = *reinterpret_cast<const uint2*>(sF + (f + 1) * LD + lane * 4);
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
        FVec<4> x;
        x.v[0] = a.x * apply_scale;
        x.v[1] = a.y * apply_scale;
        x.v[2] = b.x * apply_scale;
        x.v[3] = b.y * apply_scale;
        red_add_f32<4>(reinterpret_cast<float*>(row) + lane * 4, x);
      }
      row_cur = row_next;
    }
    __syncwarp();  // all lanes are done with buffer `cur` before the next iteration refills it
    if (done_counters != nullptr && lane == 0) {
      // streamed push: tell the copy kernel that this sample's staged rows are complete
      __threadfence();
      atomicAdd(done_counters + s / chunk_rows, 1u);
    }
  }
  cp_async_wait_group<0>();
  sync_tail(sync);  // every gradient piece of this rank is on its way to its owner
}

template <int D>
__global__ void __launch_bounds__(kWarps * 32)
interact_bwd_v2_kernel(const bf16* __restrict__ bottom, int64_t bottom_stride,
                       const bf16* __restrict__ emb, int64_t emb_stride, int n_emb,
                       const bf16* __restrict__ dz, int64_t dz_stride, bf16* __restrict__ dbottom,
                       int64_t dbottom_stride, bf16* __restrict__ demb, int64_t demb_stride,
                       float emb_grad_scale, int64_t batch,
                       const GradRoute* __restrict__ routes, int n_routes,
                       const __grid_constant__ SyncArgs sync, uint32_t* __restrict__ done_counters,
                       int chunk_rows) {
  interact_bwd_v2_body<D, kWarps, false>(bottom, bottom_stride, emb, emb_stride, n_emb, dz, dz_stride,
                                 dbottom, dbottom_stride, demb, demb_stride, emb_grad_scale, batch,
                                 routes, n_routes, sync, done_counters, chunk_rows,
                                 InteractApply{});
}

// v2 with the table update of the features in `apply` (single-GPU SGD step)
template <int D>
__global__ void __launch_bounds__(kApplyWarps * 32)
interact_bwd_apply_kernel(const bf16* __restrict__ bottom, int64_t bottom_stride,
                          const bf16* __restrict__ emb, int64_t emb_stride, int n_emb,
                          const bf16* __restrict__ dz, int64_t dz_stride,
                          bf16* __restrict__ dbottom, int64_t dbottom_stride,
                          bf16* __restrict__ demb, int64_t demb_stride, float emb_grad_scale,
                          int64_t batch, const GradRoute* __restrict__ routes, int n_routes,
                          const __grid_constant__ SyncArgs sync,
                          const __grid_constant__ InteractApply apply) {
  interact_bwd_v2_body<D, kApplyWarps, true>(bottom, bottom_stride, emb, emb_stride, n_emb, dz, dz_stride,
                                dbottom, dbottom_stride, demb, demb_stride, emb_grad_scale, batch,
                                routes, n_routes, sync, nullptr, 0, apply);
}

// dy <- dy * (y > 0) (in place) ; db[c] += sum_rows dy   (db fp32, pre-zeroed)
// Each thread owns 8 columns (one 16-byte vector) and keeps 4 rows in flight; partial column sums
// are reduced across the block in shared memory, then one atomic per column per block.
constexpr int kRbUnroll = 4;
__global__ void __launch_bounds__(256)
relu_bwd_bias_kernel(bf16* __restrict__ dy, const bf16* __restrict__ y, float* __restrict__ db,
                     int64_t rows, int cols, int rows_per_block) {
  extern __shared__ float s_part[];  // [rows_par][cols]
  const int tpr = cols >> 3;                // threads per row
  const int rows_par = blockDim.x / tpr;    // rows processed concurrently
  const int tr = threadIdx.x / tpr, tc = threadIdx.x - tr * tpr;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (tr < rows_par) {
    for (int64_t r = r0 + tr; r < r1; r += static_cast<int64_t>(rows_par) * kRbUnroll) {
      uint4 g[kRbUnroll], a[kRbUnroll];
#pragma unroll
      for (int u = 0; u < kRbUnroll; ++u) {
        const int64_t rr = r + static_cast<int64_t>(u) * rows_par;
        if (rr < r1) {
          g[u] = *reinterpret_cast<const uint4*>(dy + rr * cols + tc * 8);
          a[u] = *reinterpret_cast<const uint4*>(y + rr * cols + tc * 8);
        }
      }
#pragma unroll
      for (int u = 0; u < kRbUnroll; ++u) {
        const int64_t rr = r + static_cast<int64_t>(u) * rows_par;
        if (rr < r1) {
          uint32_t* gw = reinterpret_cast<uint32_t*>(&g[u]);
          const uint32_t* aw = reinterpret_cast<const uint32_t*>(&a[u]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float2 gf = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&gw[i]));
            const float2 af = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[i]));
            gf.x = af.x > 0.f ? gf.x : 0.f;
            gf.y = af.y > 0.f ? gf.y : 0.f;
            acc[2 * i] += gf.x;
            acc[2 * i + 1] += gf.y;
            __nv_bfloat162 h = __floats2bfloat162_rn(gf.x, gf.y);
            gw[i] = *reinterpret_cast<uint32_t*>(&h);
          }
          *reinterpret_cast<uint4*>(dy + rr * cols + tc * 8) = g[u];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_part[tr * cols + tc * 8 + i] = acc[i];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float v = 0.f;
    for (int t = 0; t < rows_par; ++t) v += s_part[t * cols + c];
    atomicAdd(db + c, v);
  }
}

// ---- low-rank cross network (DLRM-DCNv2): the element-wise parts of a layer ------------------
// x_{l+1} = x0 * s_l + x_l with s_l = W_l (V_l x_l) + b_l (the GEMMs run on cuBLASLt).  All
// tensors are [rows, D] bf16 with D a multiple of 8; each thread moves 16-byte vectors of 8
// columns and does its math in fp32, rounding once per stored element.
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = unpack2<bf16>(w[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = pack2<bf16>(f[2 * i], f[2 * i + 1]);
  return v;
}

// out = x0 * s + xl (one fma per element); flat grid-stride over 8-column vectors
__global__ void __launch_bounds__(256)
cross_fwd_kernel(const uint4* __restrict__ x0, const uint4* __restrict__ s,
                 const uint4* __restrict__ xl, uint4* __restrict__ out, int64_t n_vec) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float a[8], b[8], c[8];
    unpack8(x0[i], a);
    unpack8(s[i], b);
    unpack8(xl[i], c);
#pragma unroll
    for (int k = 0; k < 8; ++k) c[k] = fmaf(a[k], b[k], c[k]);
    out[i] = pack8(c);
  }
}

// The row-tiled kernels below split the D / 8 vector columns of a row into `n_tiles` tiles of
// `tile` vectors (blockIdx.y), so that rows of any width fit a 256-thread block the way
// relu_bwd_bias lays them out: rows_par = 256 / tile rows in flight, kRbUnroll rows per thread
// and iteration, rows_per_block rows per block (blockIdx.x).

// g = bf16(dy * x0) ; db[c] += sum_rows dy * x0 (fp32 products; per-block partial sums reduced
// in shared memory, then one atomic per column per block)
__global__ void __launch_bounds__(256)
cross_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x0, bf16* __restrict__ g,
                 float* __restrict__ db, int64_t rows, int cols, int tile, int rows_per_block) {
  extern __shared__ float s_part[];  // [rows_par][tile * 8]
  const int tpr = cols >> 3;
  const int v0 = blockIdx.y * tile;                // first vector column of this tile
  const int tw = min(tile, tpr - v0);              // vector columns in this tile
  const int rows_par = blockDim.x / tile;
  const int tr = threadIdx.x / tile, tc = threadIdx.x - tr * tile;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const bool active = tr < rows_par && tc < tw;
  if (active) {
    const int64_t col = static_cast<int64_t>(v0 + tc) * 8;
    for (int64_t r = r0 + tr; r < r1; r += static_cast<int64_t>(rows_par) * kRbUnroll) {
      uint4 a[kRbUnroll], b[kRbUnroll];
#pragma unroll
      for (int u = 0; u < kRbUnroll; ++u) {
        const int64_t rr = r + static_cast<int64_t>(u) * rows_par;
        if (rr < r1) {
          a[u] = *reinterpret_cast<const uint4*>(dy + rr * cols + col);
          b[u] = *reinterpret_cast<const uint4*>(x0 + rr * cols + col);
        }
      }
#pragma unroll
      for (int u = 0; u < kRbUnroll; ++u) {
        const int64_t rr = r + static_cast<int64_t>(u) * rows_par;
        if (rr < r1) {
          float fa[8], fb[8];
          unpack8(a[u], fa);
          unpack8(b[u], fb);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            fa[k] *= fb[k];
            acc[k] += fa[k];
          }
          *reinterpret_cast<uint4*>(g + rr * cols + col) = pack8(fa);
        }
      }
    }
  }
  if (tr < rows_par) {
#pragma unroll
    for (int k = 0; k < 8; ++k) s_part[tr * tile * 8 + tc * 8 + k] = acc[k];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < tw * 8; c += blockDim.x) {
    float v = 0.f;
    for (int t = 0; t < rows_par; ++t) v += s_part[t * tile * 8 + c];
    atomicAdd(db + v0 * 8 + c, v);
  }
}

// dx0 = d_chain + sum_l dy_l * s_l (fp32, rounded once).  Columns below emb_cols go to dx0, the
// others (the bottom-MLP vector) to the contiguous d_bottom [rows, cols - emb_cols].
__global__ void __launch_bounds__(256)
cross_dx0_kernel(const bf16* __restrict__ d_chain, const __grid_constant__ CrossTerms terms,
                 bf16* __restrict__ dx0, bf16* __restrict__ d_bottom, int64_t rows, int cols,
                 int emb_cols, int tile, int rows_per_block) {
  const int tpr = cols >> 3;
  const int v0 = blockIdx.y * tile;
  const int tw = min(tile, tpr - v0);
  const int rows_par = blockDim.x / tile;
  const int tr = threadIdx.x / tile, tc = threadIdx.x - tr * tile;
  if (tr >= rows_par || tc >= tw) return;
  const int col = (v0 + tc) * 8;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  const int bcols = cols - emb_cols;
  bf16* dst = col < emb_cols ? dx0 + col : d_bottom + (col - emb_cols);
  const int64_t dst_stride = col < emb_cols ? cols : bcols;
  for (int64_t r = r0 + tr; r < r1; r += rows_par) {
    const int64_t off = r * cols + col;
    float acc[8];
    unpack8(*reinterpret_cast<const uint4*>(d_chain + off), acc);
    for (int l = 0; l < terms.n; ++l) {
      float a[8], b[8];
      unpack8(*(reinterpret_cast<const uint4*>(terms.dy[l]) + off / 8), a);
      unpack8(*(reinterpret_cast<const uint4*>(terms.s[l]) + off / 8), b);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = fmaf(a[k], b[k], acc[k]);
    }
    *reinterpret_cast<uint4*>(dst + r * dst_stride) = pack8(acc);
  }
}

// Final layer (K -> 1) + BCE-with-logits loss + backward of both, one warp per sample:
//   logit = <x, w> + b ; loss += softplus terms ; dlogit = (sigmoid(logit) - label) * inv_batch
//   dx = dlogit * w masked by (x > 0) (x is a ReLU output) ; dw += dlogit * x ; db += dlogit ;
//   dbias_prev[c] += dx[c]  (bias gradient of the layer that produced x)
template <int PL>
__global__ void __launch_bounds__(256)
head_loss_kernel(const bf16* __restrict__ x, int K, const bf16* __restrict__ w,
                 const bf16* __restrict__ bias, const float* __restrict__ labels, int64_t batch,
                 float inv_batch, bf16* __restrict__ dx, float* __restrict__ dw,
                 float* __restrict__ db, float* __restrict__ dbias_prev,
                 float* __restrict__ loss_sum, float* __restrict__ logits_out) {
  extern __shared__ float sred[];  // [2 * K + 2] per block: dw partial, dbias_prev partial
  float* s_dw = sred;
  float* s_dbp = sred + K;
  float* s_misc = sred + 2 * K;  // [0] loss, [1] db
  for (int i = threadIdx.x; i < 2 * K + 2; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  constexpr int per_lane = PL;  // K == 32 * PL
  const float b0 = __bfloat162float(bias[0]);
  float wreg[PL];
#pragma unroll
  for (int i = 0; i < PL; ++i) wreg[i] = __bfloat162float(w[lane + 32 * i]);
  float dw_acc[PL], dbp_acc[PL];
#pragma unroll
  for (int i = 0; i < PL; ++i) dw_acc[i] = dbp_acc[i] = 0.f;
  float loss_acc = 0.f, db_acc = 0.f;
  for (int64_t s = static_cast<int64_t>(blockIdx.x) * wpb + warp; s < batch;
       s += static_cast<int64_t>(gridDim.x) * wpb) {
    float xv[PL];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      if (i < per_lane) {
        xv[i] = __bfloat162float(x[s * K + lane + 32 * i]);
        dot = fmaf(xv[i], wreg[i], dot);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
    const float logit = dot + b0;
    const float label = labels[s];
    // numerically stable BCE with logits
    const float loss = fmaxf(logit, 0.f) - logit * label + log1pf(__expf(-fabsf(logit)));
    const float sig = 1.f / (1.f + __expf(-logit));
    const float dl = (sig - label) * inv_batch;
    if (lane == 0) {
      loss_acc += loss;
      db_acc += dl;
      if (logits_out) logits_out[s] = logit;
    }
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      if (i < per_lane) {
        dw_acc[i] = fmaf(dl, xv[i], dw_acc[i]);
        const float g = xv[i] > 0.f ? dl * wreg[i] : 0.f;
        dbp_acc[i] += g;
        dx[s * K + lane + 32 * i] = __float2bfloat16_rn(g);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < PL; ++i) {
    if (i < per_lane) {
      atomicAdd(&s_dw[lane + 32 * i], dw_acc[i]);
      atomicAdd(&s_dbp[lane + 32 * i], dbp_acc[i]);
    }
  }
  if (lane == 0) {
    atomicAdd(&s_misc[0], loss_acc);
    atomicAdd(&s_misc[1], db_acc);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    atomicAdd(dw + i, s_dw[i]);
    atomicAdd(dbias_prev + i, s_dbp[i]);
  }
  if (threadIdx.x == 0) {
    atomicAdd(loss_sum, s_misc[0] * inv_batch);
    atomicAdd(db, s_misc[1]);
  }
}

// Forward-only counterpart of head_loss_kernel (evaluation).  Each warp takes groups of 32
// samples; every sample's logit is computed by the whole warp exactly as head_loss computes it
// (lane-strided fmaf, the same shuffle reduction, bias added last), so the logits are bit
// identical, and lane j keeps the logit of sample j of the group.  Per sample:
//   probs[s] = sigmoid(logit)                                    (every row s < batch)
//   rows s < *n_valid only: hist[label > 0.5][k(p)] += 1, loss_sum += BCE-with-logits, count += 1
// with k(p) = clamp(ceil(fp32(p * nb)) - 1, 0, nb - 1), nb = hist columns (utils/metrics.py,
// BinnedAUC).  Histogram adds are warp aggregated: one atomic per distinct bucket per group.
template <int PL>
__global__ void __launch_bounds__(256)
head_eval_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                 const bf16* __restrict__ bias, const float* __restrict__ labels, int64_t batch,
                 const int64_t* __restrict__ n_valid, float* __restrict__ probs,
                 unsigned long long* __restrict__ hist, int nb, double* __restrict__ loss_sum,
                 unsigned long long* __restrict__ count) {
  constexpr int K = 32 * PL;
  __shared__ float s_loss;
  if (threadIdx.x == 0) s_loss = 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  int64_t nv = *n_valid;
  nv = nv < 0 ? 0 : (nv > batch ? batch : nv);
  const float b0 = __bfloat162float(bias[0]);
  const float nbf = static_cast<float>(nb);
  float wreg[PL];
#pragma unroll
  for (int i = 0; i < PL; ++i) wreg[i] = __bfloat162float(w[lane + 32 * i]);
  float loss_acc = 0.f;
  for (int64_t g0 = (static_cast<int64_t>(blockIdx.x) * wpb + warp) * 32; g0 < batch;
       g0 += static_cast<int64_t>(gridDim.x) * wpb * 32) {
    const int rows = batch - g0 < 32 ? static_cast<int>(batch - g0) : 32;
    float my_logit = 0.f;
#pragma unroll 4
    for (int j = 0; j < rows; ++j) {
      const bf16* xr = x + (g0 + j) * K;
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < PL; ++i) dot = fmaf(__bfloat162float(xr[lane + 32 * i]), wreg[i], dot);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
      if (lane == j) my_logit = dot + b0;
    }
    const int64_t s = g0 + lane;
    const bool has_row = lane < rows;
    const bool valid = s < nv;  // implies has_row
    const float logit = my_logit;
    const float p = 1.f / (1.f + __expf(-logit));
    if (has_row) probs[s] = p;
    int key = -1;
    if (valid) {
      const float label = labels[s];
      loss_acc += fmaxf(logit, 0.f) - logit * label + log1pf(__expf(-fabsf(logit)));
      int k = static_cast<int>(ceilf(__fmul_rn(p, nbf))) - 1;
      k = k < 0 ? 0 : (k > nb - 1 ? nb - 1 : k);
      key = (label > 0.5f ? nb : 0) + k;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && lane == __ffs(peers) - 1)
      atomicAdd(hist + key, static_cast<unsigned long long>(__popc(peers)));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
  if (lane == 0) atomicAdd(&s_loss, loss_acc);
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(loss_sum, static_cast<double>(s_loss));
    if (blockIdx.x == 0) atomicAdd(count, static_cast<unsigned long long>(nv));
  }
}

// p32 -= lr * g32 ; p16 = bf16(p32) ; g32 = 0   (lr read from device memory: graph replay safe)
// kDecay: p32 -= lr * (grad_scale * g32 + weight_decay * p32), SGD's update under either weight
// decay mode
template <bool kDecay>
__global__ void __launch_bounds__(256)
sgd_update_kernel(float* __restrict__ p32, bf16* __restrict__ p16, float* __restrict__ g32,
                  const float* __restrict__ lr_ptr, float grad_scale, float weight_decay,
                  int64_t n_vec4) {
  const float step = -(*lr_ptr) * grad_scale;
  const float neg_lr = -(*lr_ptr);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec4;
       i += stride) {
    float4 p = reinterpret_cast<float4*>(p32)[i];
    const float4 g = reinterpret_cast<const float4*>(g32)[i];
    if constexpr (kDecay) {
      p.x = fmaf(neg_lr, fmaf(weight_decay, p.x, __fmul_rn(grad_scale, g.x)), p.x);
      p.y = fmaf(neg_lr, fmaf(weight_decay, p.y, __fmul_rn(grad_scale, g.y)), p.y);
      p.z = fmaf(neg_lr, fmaf(weight_decay, p.z, __fmul_rn(grad_scale, g.z)), p.z);
      p.w = fmaf(neg_lr, fmaf(weight_decay, p.w, __fmul_rn(grad_scale, g.w)), p.w);
    } else {
      p.x = fmaf(step, g.x, p.x);
      p.y = fmaf(step, g.y, p.y);
      p.z = fmaf(step, g.z, p.z);
      p.w = fmaf(step, g.w, p.w);
    }
    reinterpret_cast<float4*>(p32)[i] = p;
    reinterpret_cast<float4*>(g32)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __nv_bfloat162 a = __floats2bfloat162_rn(p.x, p.y), b = __floats2bfloat162_rn(p.z, p.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&a);
    o.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(p16)[i] = o;
  }
}

// Adagrad / Adam over the flat dense buffers, element by element with the expressions of the
// embedding update (apply_update in sparse_update_kernels.cu), then p16 = bf16(p32) and g32 = 0
// (the next step's gradient kernels accumulate into g32).  lr and Adam's step count t are device
// words: graph replay safe.  s0 = Adagrad accumulator or Adam m, s1 = Adam v.  DECAY: 0 none,
// kDenseDecayL2 (g += weight_decay * p before the update), kDenseDecayDecoupled (p *= 1 - lr *
// weight_decay before the step, which the undecayed g drives: torch.optim.AdamW's order).
constexpr int kDenseDecayL2 = 1;
constexpr int kDenseDecayDecoupled = 2;

template <int KIND, int DECAY>
__device__ __forceinline__ void dense_opt_elem(float& p, float& a, float& v, float g, float lr,
                                               float beta1, float beta2, float bias1, float bias2,
                                               float eps, float weight_decay, float keep) {
  if constexpr (DECAY == kDenseDecayL2) g = fmaf(weight_decay, p, g);
  if constexpr (DECAY == kDenseDecayDecoupled) p = __fmul_rn(p, keep);
  if constexpr (KIND == kOptAdagrad) {
    a = fmaf(g, g, a);
    p -= lr * g / (sqrtf(a) + eps);
  } else {
    a = beta1 * a + (1.f - beta1) * g;
    v = beta2 * v + (1.f - beta2) * g * g;
    const float mh = a / bias1;
    const float vh = v / bias2;
    p -= lr * mh / (sqrtf(vh) + eps);
  }
}

template <int KIND, int DECAY>
__global__ void __launch_bounds__(256)
dense_opt_kernel(float* __restrict__ p32, bf16* __restrict__ p16, float* __restrict__ g32,
                 float* __restrict__ s0, float* __restrict__ s1, const float* __restrict__ lr_ptr,
                 const float* __restrict__ step_ptr, float beta1, float beta2, float eps,
                 float weight_decay, int64_t n_vec4) {
  const float lr = *lr_ptr;
  const float keep = fmaf(-lr, weight_decay, 1.f);  // decoupled decay only
  float bias1 = 1.f, bias2 = 1.f;
  if constexpr (KIND == kOptAdam) {  // bias corrections as resolve_step computes them
    const float t = *step_ptr;
    bias1 = 1.f - powf(beta1, t);
    bias2 = 1.f - powf(beta2, t);
  }
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec4;
       i += stride) {
    float4 p = reinterpret_cast<float4*>(p32)[i];
    const float4 g = reinterpret_cast<const float4*>(g32)[i];
    float4 a = reinterpret_cast<float4*>(s0)[i];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (KIND == kOptAdam) v = reinterpret_cast<float4*>(s1)[i];
    dense_opt_elem<KIND, DECAY>(p.x, a.x, v.x, g.x, lr, beta1, beta2, bias1, bias2, eps,
                                weight_decay, keep);
    dense_opt_elem<KIND, DECAY>(p.y, a.y, v.y, g.y, lr, beta1, beta2, bias1, bias2, eps,
                                weight_decay, keep);
    dense_opt_elem<KIND, DECAY>(p.z, a.z, v.z, g.z, lr, beta1, beta2, bias1, bias2, eps,
                                weight_decay, keep);
    dense_opt_elem<KIND, DECAY>(p.w, a.w, v.w, g.w, lr, beta1, beta2, bias1, bias2, eps,
                                weight_decay, keep);
    reinterpret_cast<float4*>(p32)[i] = p;
    reinterpret_cast<float4*>(s0)[i] = a;
    if constexpr (KIND == kOptAdam) reinterpret_cast<float4*>(s1)[i] = v;
    reinterpret_cast<float4*>(g32)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    reinterpret_cast<uint2*>(p16)[i] = o;
  }
}

// Momentum SGD over the flat dense buffers with the expressions of the embedding update
// (kOptMomentum in apply_update): b = fmaf(mu, b, g), p = fmaf(-lr, b, p) or, NESTEROV,
// p = fmaf(-lr, fmaf(mu, b, g), p); then p16 = bf16(p32) and g32 = 0.  DECAY as dense_opt_kernel.
template <int DECAY, bool NESTEROV>
__device__ __forceinline__ void dense_momentum_elem(float& p, float& b, float g, float neg_lr,
                                                    float mu, float weight_decay, float keep) {
  if constexpr (DECAY == kDenseDecayL2) g = fmaf(weight_decay, p, g);
  if constexpr (DECAY == kDenseDecayDecoupled) p = __fmul_rn(p, keep);
  b = fmaf(mu, b, g);
  p = fmaf(neg_lr, NESTEROV ? fmaf(mu, b, g) : b, p);
}

template <int DECAY, bool NESTEROV>
__global__ void __launch_bounds__(256)
dense_momentum_kernel(float* __restrict__ p32, bf16* __restrict__ p16, float* __restrict__ g32,
                      float* __restrict__ buf, const float* __restrict__ lr_ptr, float mu,
                      float weight_decay, int64_t n_vec4) {
  const float lr = *lr_ptr;
  const float keep = fmaf(-lr, weight_decay, 1.f);  // decoupled decay only
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec4;
       i += stride) {
    float4 p = reinterpret_cast<float4*>(p32)[i];
    const float4 g = reinterpret_cast<const float4*>(g32)[i];
    float4 b = reinterpret_cast<float4*>(buf)[i];
    dense_momentum_elem<DECAY, NESTEROV>(p.x, b.x, g.x, -lr, mu, weight_decay, keep);
    dense_momentum_elem<DECAY, NESTEROV>(p.y, b.y, g.y, -lr, mu, weight_decay, keep);
    dense_momentum_elem<DECAY, NESTEROV>(p.z, b.z, g.z, -lr, mu, weight_decay, keep);
    dense_momentum_elem<DECAY, NESTEROV>(p.w, b.w, g.w, -lr, mu, weight_decay, keep);
    reinterpret_cast<float4*>(p32)[i] = p;
    reinterpret_cast<float4*>(buf)[i] = b;
    reinterpret_cast<float4*>(g32)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    reinterpret_cast<uint2*>(p16)[i] = o;
  }
}

// dst[r, 0:dst_cols] = bf16(src[r, 0:src_cols]) zero padded
__global__ void cast_pad_kernel(const float* __restrict__ src, int src_cols, bf16* __restrict__ dst,
                                int dst_cols, int64_t rows) {
  const int64_t n = rows * dst_cols;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    const int64_t r = i / dst_cols;
    const int c = static_cast<int>(i - r * dst_cols);
    dst[i] = __float2bfloat16_rn(c < src_cols ? src[r * src_cols + c] : 0.f);
  }
}

// ---- 1-D average pooling over the concatenated embeddings ("same" padding, partial windows
// divide by the number of real elements): the memory-bound stand-in for FM / pooling
// interactions in the synthetic models (reference synthetic_models.py:150-160, Keras
// AveragePooling1D).  out[r, j] = mean(x[r, j*stride-left : (j+1)*stride-left] ∩ [0, n)).
__global__ void __launch_bounds__(256)
avgpool_fwd_kernel(const bf16* __restrict__ x, int64_t x_stride, int n, bf16* __restrict__ out,
                   int64_t out_stride, int out_len, int stride, int left, int64_t rows) {
  const int64_t total = rows * out_len;
  const int64_t step = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += step) {
    const int64_t r = i / out_len;
    const int j = static_cast<int>(i - r * out_len);
    const int lo = max(0, j * stride - left), hi = min(n, (j + 1) * stride - left);
    const bf16* xp = x + r * x_stride;
    float acc = 0.f;
    for (int c = lo; c < hi; ++c) acc += __bfloat162float(xp[c]);
    out[r * out_stride + j] = __float2bfloat16_rn(hi > lo ? acc / static_cast<float>(hi - lo) : 0.f);
  }
}

// dx[r, c] = dout[r, window(c)] / count(window(c))
__global__ void __launch_bounds__(256)
avgpool_bwd_kernel(const bf16* __restrict__ dout, int64_t dout_stride, int out_len,
                   bf16* __restrict__ dx, int64_t dx_stride, int n, int stride, int left,
                   int64_t rows) {
  const int64_t total = rows * n;
  const int64_t step = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += step) {
    const int64_t r = i / n;
    const int c = static_cast<int>(i - r * n);
    const int j = (c + left) / stride;
    const int lo = max(0, j * stride - left), hi = min(n, (j + 1) * stride - left);
    const float g = j < out_len ? __bfloat162float(dout[r * dout_stride + j]) : 0.f;
    dx[r * dx_stride + c] = __float2bfloat16_rn(g / static_cast<float>(hi - lo));
  }
}

}  // namespace

void launch_avgpool_fwd(const void* x, int64_t x_stride, int n, void* out, int64_t out_stride,
                        int out_len, int stride, int left, int64_t rows, cudaStream_t stream) {
  if (rows <= 0 || out_len <= 0) return;
  int64_t blocks = (rows * out_len + 255) / 256;
  if (blocks > kGridCapSms * 16) blocks = kGridCapSms * 16;
  avgpool_fwd_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(x), x_stride, n, reinterpret_cast<bf16*>(out), out_stride,
      out_len, stride, left, rows);
}

void launch_avgpool_bwd(const void* dout, int64_t dout_stride, int out_len, void* dx,
                        int64_t dx_stride, int n, int stride, int left, int64_t rows,
                        cudaStream_t stream) {
  if (rows <= 0 || n <= 0) return;
  int64_t blocks = (rows * n + 255) / 256;
  if (blocks > kGridCapSms * 16) blocks = kGridCapSms * 16;
  avgpool_bwd_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(dout), dout_stride, out_len, reinterpret_cast<bf16*>(dx),
      dx_stride, n, stride, left, rows);
}

bool launch_interact_fwd(const void* bottom, int64_t bottom_stride, const void* emb,
                         int64_t emb_stride, int n_emb, int dim, void* z, int64_t z_stride,
                         int z_width, int64_t batch, int sm_count, cudaStream_t stream,
                         const SyncArgs& sync) {
  if (n_emb + 1 > kMaxFeat || batch <= 0) return false;
#define DE_IFWD(DD)                                                                              \
  {                                                                                              \
    const int smem = fwd_head_bytes(DD) + kWarps * fwd_warp_bytes(DD, n_emb);                   \
    cudaFuncSetAttribute(interact_fwd_kernel<DD>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                         smem);                                                                  \
    int per_sm = 0;                                                                              \
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, interact_fwd_kernel<DD>, kWarps * 32, \
                                                  smem);                                         \
    int64_t blocks = (batch + kWarps - 1) / kWarps;                                              \
    const int64_t cap = static_cast<int64_t>(sm_count) * (per_sm > 0 ? per_sm : 1);              \
    if (blocks > cap) blocks = cap;                                                              \
    interact_fwd_kernel<DD><<<static_cast<unsigned>(blocks), kWarps * 32, smem, stream>>>(       \
        reinterpret_cast<const bf16*>(bottom), bottom_stride, reinterpret_cast<const bf16*>(emb), \
        emb_stride, n_emb, reinterpret_cast<bf16*>(z), z_stride, z_width, batch, sync);          \
    return true;                                                                                 \
  }
  if (dim == 128) DE_IFWD(128)
  if (dim == 64) DE_IFWD(64)
  if (dim == 32) DE_IFWD(32)
  if (dim == 16) DE_IFWD(16)
#undef DE_IFWD
  return false;
}

bool launch_interact_bwd(const void* bottom, int64_t bottom_stride, const void* emb,
                         int64_t emb_stride, int n_emb, int dim, const void* dz,
                         int64_t dz_stride, void* dbottom, int64_t dbottom_stride, void* demb,
                         int64_t demb_stride, float emb_grad_scale, int64_t batch, int sm_count,
                         cudaStream_t stream, const GradRoute* routes, int n_routes,
                         const SyncArgs& sync, uint32_t* done_counters, int chunk_rows,
                         const InteractApply* apply) {
  if (n_emb + 1 > kMaxFeat || batch <= 0 || dim % 32 != 0) return false;
  const bool applied = apply != nullptr && apply->mask != 0;
  if (applied && (dim != 128 || done_counters != nullptr)) return false;
  int64_t blocks = (batch + kWarps - 1) / kWarps;
  const int64_t cap = static_cast<int64_t>(sm_count) * 8;
  if (blocks > cap) blocks = cap;
  // DE_B200_INTERACT_V1=1 selects the single-buffered kernel (local gradient buffer only)
  static const bool force_v1 = [] {
    const char* v = std::getenv("DE_B200_INTERACT_V1");
    return v != nullptr && v[0] == '1';
  }();
  const int nf = n_emb + 1;
  const int dz_elems = (nf * (nf - 1) / 2 + dim + 7) / 8 * 8;
  const bool v2_ok =
      dz_elems <= kDzMax && dz_elems <= dz_stride && dz_stride % 8 == 0 &&
      bottom_stride % 8 == 0 && emb_stride % 8 == 0 && dbottom_stride % 8 == 0 &&
      ((reinterpret_cast<uintptr_t>(dz) | reinterpret_cast<uintptr_t>(bottom) |
        reinterpret_cast<uintptr_t>(emb) | reinterpret_cast<uintptr_t>(dbottom)) & 15) == 0 &&
      (dim == 128 || dim == 64) &&
      (routes != nullptr || (demb_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(demb) & 15) == 0));
  if ((routes != nullptr || done_counters != nullptr || applied) && !v2_ok) return false;  // v2 only
  const bool has_sync = sync.state != nullptr && (sync.wait_ch >= 0 || sync.signal_ch >= 0);
  if (v2_ok &&
      (!force_v1 || routes != nullptr || has_sync || done_counters != nullptr || applied)) {
    // as many resident blocks per SM as the shared memory of n_emb allows, each warp streams its
    // samples through a double buffer
#define DE_IBWD2(KERNEL, DD, W, ...)                                                             \
  {                                                                                              \
    const int smem = bwd_head_bytes(DD) + W * bwd_warp_bytes(DD, n_emb) +                        \
                     n_emb * (DD / 8) * static_cast<int>(sizeof(ChunkDst));                      \
    cudaFuncSetAttribute(KERNEL<DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);         \
    int per_sm = 0;                                                                              \
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, KERNEL<DD>, W * 32, smem);            \
    int64_t blocks2 = (batch + W - 1) / W;                                                       \
    const int64_t cap2 = static_cast<int64_t>(sm_count) * (per_sm > 0 ? per_sm : 1);             \
    if (blocks2 > cap2) blocks2 = cap2;                                                          \
    KERNEL<DD><<<static_cast<unsigned>(blocks2), W * 32, smem, stream>>>(                        \
        reinterpret_cast<const bf16*>(bottom), bottom_stride, reinterpret_cast<const bf16*>(emb), \
        emb_stride, n_emb, reinterpret_cast<const bf16*>(dz), dz_stride,                         \
        reinterpret_cast<bf16*>(dbottom), dbottom_stride, reinterpret_cast<bf16*>(demb),         \
        demb_stride, emb_grad_scale, batch, routes, n_routes, sync, __VA_ARGS__);                \
    return true;                                                                                 \
  }
    if (applied) DE_IBWD2(interact_bwd_apply_kernel, 128, kApplyWarps, *apply)
    if (dim == 128) DE_IBWD2(interact_bwd_v2_kernel, 128, kWarps, done_counters, chunk_rows)
    if (dim == 64) DE_IBWD2(interact_bwd_v2_kernel, 64, kWarps, done_counters, chunk_rows)
#undef DE_IBWD2
  }
  if (has_sync) return false;
#define DE_IBWD(DD)                                                                              \
  {                                                                                              \
    const size_t smem = kWarps * (kMaxFeat * (DD + 8) + kMaxFeat * 40) * sizeof(bf16);           \
    cudaFuncSetAttribute(interact_bwd_kernel<DD>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                         static_cast<int>(smem));                                                \
    interact_bwd_kernel<DD><<<static_cast<unsigned>(blocks), kWarps * 32, smem, stream>>>(       \
        reinterpret_cast<const bf16*>(bottom), bottom_stride, reinterpret_cast<const bf16*>(emb), \
        emb_stride, n_emb, reinterpret_cast<const bf16*>(dz), dz_stride,                         \
        reinterpret_cast<bf16*>(dbottom), dbottom_stride, reinterpret_cast<bf16*>(demb),         \
        demb_stride, emb_grad_scale, batch);                                                     \
    return true;                                                                                 \
  }
  if (dim == 128) DE_IBWD(128)
  if (dim == 64) DE_IBWD(64)
  if (dim == 32) DE_IBWD(32)
#undef DE_IBWD
  return false;
}

// Tiling of the row-tiled cross kernels: the number of column tiles that keeps the most of a
// 256-thread block busy (each tile holds at most 256 vector columns).
static void cross_tiling(int cols, int* tile, int* n_tiles, int* rows_per_block) {
  const int tpr = cols / 8;
  int best_t = 0, best_n = 0;
  double best = -1.0;
  for (int n = (tpr + 255) / 256; n <= tpr && n <= 64; ++n) {
    const int t = (tpr + n - 1) / n;
    const int rows_par = 256 / t;
    const double busy = static_cast<double>(rows_par * t) / 256.0 *
                        static_cast<double>(tpr) / static_cast<double>(n * t);
    if (busy > best + 1e-9) {
      best = busy;
      best_t = t;
      best_n = n;
    }
  }
  *tile = best_t;
  *n_tiles = best_n;
  // ~16 rows per thread, as relu_bwd_bias
  *rows_per_block = (256 / best_t) * kRbUnroll * 4;
}

void launch_cross_fwd(const void* x0, const void* s, const void* xl, void* out, int64_t n,
                      int sm_count, cudaStream_t stream) {
  const int64_t n_vec = n / 8;
  if (n_vec <= 0) return;
  int64_t blocks = (n_vec + 255) / 256;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  cross_fwd_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(x0), reinterpret_cast<const uint4*>(s),
      reinterpret_cast<const uint4*>(xl), reinterpret_cast<uint4*>(out), n_vec);
}

void launch_cross_bwd(const void* dy, const void* x0, void* g, float* db, int64_t rows, int cols,
                      cudaStream_t stream) {
  if (rows <= 0) return;
  int tile, n_tiles, rpb;
  cross_tiling(cols, &tile, &n_tiles, &rpb);
  const dim3 grid(static_cast<unsigned>((rows + rpb - 1) / rpb), static_cast<unsigned>(n_tiles));
  const size_t smem = static_cast<size_t>(256 / tile) * tile * 8 * sizeof(float);
  cross_bwd_kernel<<<grid, 256, smem, stream>>>(
      reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x0),
      reinterpret_cast<bf16*>(g), db, rows, cols, tile, rpb);
}

void launch_cross_dx0(const void* d_chain, const CrossTerms& terms, void* dx0, void* d_bottom,
                      int64_t rows, int cols, int emb_cols, cudaStream_t stream) {
  if (rows <= 0) return;
  int tile, n_tiles, rpb;
  cross_tiling(cols, &tile, &n_tiles, &rpb);
  const dim3 grid(static_cast<unsigned>((rows + rpb - 1) / rpb), static_cast<unsigned>(n_tiles));
  cross_dx0_kernel<<<grid, 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(d_chain), terms, reinterpret_cast<bf16*>(dx0),
      reinterpret_cast<bf16*>(d_bottom), rows, cols, emb_cols, tile, rpb);
}

void launch_relu_bwd_bias(void* dy, const void* y, float* db, int64_t rows, int cols,
                          cudaStream_t stream) {
  if (rows <= 0) return;
  const int tpr = cols / 8;
  const int threads = 256;  // cols <= 2048
  const int rows_par = threads / tpr;
  // ~16 rows per thread (4 batches of 4 in flight); >= 2048 blocks at batch 64k
  const int rows_per_block = rows_par * kRbUnroll * 4;
  const int64_t blocks = (rows + rows_per_block - 1) / rows_per_block;
  const size_t smem = static_cast<size_t>(rows_par) * cols * sizeof(float);
  relu_bwd_bias_kernel<<<static_cast<unsigned>(blocks), threads, smem, stream>>>(
      reinterpret_cast<bf16*>(dy), reinterpret_cast<const bf16*>(y), db, rows, cols,
      rows_per_block);
}

bool launch_head_loss(const void* x, int K, const void* w, const void* bias, const float* labels,
                      int64_t batch, float inv_batch, void* dx, float* dw, float* db,
                      float* dbias_prev, float* loss_sum, float* logits_out, int sm_count,
                      cudaStream_t stream) {
  if (batch <= 0) return true;
  const int threads = 256;
  int64_t blocks = (batch + 7) / 8;
  if (blocks > sm_count * 4) blocks = sm_count * 4;
  const size_t smem = (2 * K + 2) * sizeof(float);
#define DE_HEAD(PL)                                                                              \
  head_loss_kernel<PL><<<static_cast<unsigned>(blocks), threads, smem, stream>>>(                \
      reinterpret_cast<const bf16*>(x), K, reinterpret_cast<const bf16*>(w),                     \
      reinterpret_cast<const bf16*>(bias), labels, batch, inv_batch, reinterpret_cast<bf16*>(dx), \
      dw, db, dbias_prev, loss_sum, logits_out)
  switch (K) {
    case 64: DE_HEAD(2); break;
    case 128: DE_HEAD(4); break;
    case 256: DE_HEAD(8); break;
    case 512: DE_HEAD(16); break;
    case 1024: DE_HEAD(32); break;
    default: return false;
  }
#undef DE_HEAD
  return true;
}

bool launch_head_eval(const void* x, int K, const void* w, const void* bias, const float* labels,
                      int64_t batch, const int64_t* n_valid, float* probs, int64_t* hist, int nb,
                      double* loss_sum, int64_t* count, int sm_count, cudaStream_t stream) {
  if (K != 64 && K != 128 && K != 256 && K != 512 && K != 1024) return false;
  if (batch <= 0) return true;
  const int threads = 256;  // 8 warps, 32 samples per warp and group
  int64_t blocks = (batch + 255) / 256;
  if (blocks > sm_count * 4) blocks = sm_count * 4;
#define DE_HEAD_EVAL(PL)                                                                         \
  head_eval_kernel<PL><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(                  \
      reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(w),                        \
      reinterpret_cast<const bf16*>(bias), labels, batch, n_valid, probs,                        \
      reinterpret_cast<unsigned long long*>(hist), nb, loss_sum,                                 \
      reinterpret_cast<unsigned long long*>(count))
  switch (K) {
    case 64: DE_HEAD_EVAL(2); break;
    case 128: DE_HEAD_EVAL(4); break;
    case 256: DE_HEAD_EVAL(8); break;
    case 512: DE_HEAD_EVAL(16); break;
    default: DE_HEAD_EVAL(32); break;
  }
#undef DE_HEAD_EVAL
  return true;
}

void launch_sgd_update(float* p32, void* p16, float* g32, const float* lr_ptr, float grad_scale,
                       int64_t n, int sm_count, cudaStream_t stream, float weight_decay) {
  const int64_t n_vec4 = n / 4;  // buffers are padded to 16 bytes
  if (n_vec4 <= 0) return;
  int64_t blocks = (n_vec4 + 255) / 256;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  auto launch = [&](auto kernel) {
    kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        p32, reinterpret_cast<bf16*>(p16), g32, lr_ptr, grad_scale, weight_decay, n_vec4);
  };
  if (weight_decay != 0.f) launch(sgd_update_kernel<true>);
  else launch(sgd_update_kernel<false>);
}

bool launch_dense_opt(int kind, float* p32, void* p16, float* g32, float* s0, float* s1,
                      const float* lr_ptr, const float* step_ptr, float beta1, float beta2,
                      float eps, int64_t n, int sm_count, cudaStream_t stream, float weight_decay,
                      int weight_decay_mode) {
  if (kind != kOptAdagrad && kind != kOptAdam) return false;
  const int64_t n_vec4 = n / 4;  // buffers are padded to 16 bytes
  if (n_vec4 <= 0) return true;
  int64_t blocks = (n_vec4 + 255) / 256;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  const int decay = weight_decay == 0.f ? 0
                    : weight_decay_mode == kWeightDecayDecoupled ? kDenseDecayDecoupled
                                                                 : kDenseDecayL2;
  auto launch = [&](auto kind_c, auto decay_c) {
    constexpr int K = decltype(kind_c)::value, D = decltype(decay_c)::value;
    dense_opt_kernel<K, D><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        p32, reinterpret_cast<bf16*>(p16), g32, s0, K == kOptAdam ? s1 : nullptr, lr_ptr,
        K == kOptAdam ? step_ptr : nullptr, K == kOptAdam ? beta1 : 0.f,
        K == kOptAdam ? beta2 : 0.f, eps, weight_decay, n_vec4);
  };
  auto with_decay = [&](auto kind_c) {
    if (decay == kDenseDecayDecoupled)
      launch(kind_c, std::integral_constant<int, kDenseDecayDecoupled>{});
    else if (decay == kDenseDecayL2)
      launch(kind_c, std::integral_constant<int, kDenseDecayL2>{});
    else
      launch(kind_c, std::integral_constant<int, 0>{});
  };
  if (kind == kOptAdagrad) with_decay(std::integral_constant<int, kOptAdagrad>{});
  else with_decay(std::integral_constant<int, kOptAdam>{});
  return true;
}

void launch_dense_momentum(float* p32, void* p16, float* g32, float* b, const float* lr_ptr,
                           float momentum, bool nesterov, int64_t n, int sm_count,
                           cudaStream_t stream, float weight_decay, int weight_decay_mode) {
  const int64_t n_vec4 = n / 4;  // buffers are padded to 16 bytes
  if (n_vec4 <= 0) return;
  int64_t blocks = (n_vec4 + 255) / 256;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  const int decay = weight_decay == 0.f ? 0
                    : weight_decay_mode == kWeightDecayDecoupled ? kDenseDecayDecoupled
                                                                 : kDenseDecayL2;
  auto launch = [&](auto decay_c, auto nesterov_c) {
    dense_momentum_kernel<decltype(decay_c)::value, decltype(nesterov_c)::value>
        <<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
            p32, reinterpret_cast<bf16*>(p16), g32, b, lr_ptr, momentum, weight_decay, n_vec4);
  };
  auto with_nesterov = [&](auto decay_c) {
    if (nesterov) launch(decay_c, std::true_type{});
    else launch(decay_c, std::false_type{});
  };
  if (decay == kDenseDecayDecoupled)
    with_nesterov(std::integral_constant<int, kDenseDecayDecoupled>{});
  else if (decay == kDenseDecayL2)
    with_nesterov(std::integral_constant<int, kDenseDecayL2>{});
  else
    with_nesterov(std::integral_constant<int, 0>{});
}

void launch_cast_pad(const float* src, int src_cols, void* dst, int dst_cols, int64_t rows,
                     cudaStream_t stream) {
  if (rows <= 0) return;
  int64_t blocks = (rows * dst_cols + 255) / 256;
  if (blocks > kGridCapSms * 8) blocks = kGridCapSms * 8;
  cast_pad_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      src, src_cols, reinterpret_cast<bf16*>(dst), dst_cols, rows);
}

}  // namespace de
