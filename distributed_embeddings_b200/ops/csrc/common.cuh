// Device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "de_b200.h"

namespace de {

constexpr int64_t kSentinelKey = 0x7fffffffffffffffLL;

__host__ __device__ __forceinline__ int pow2_ceil(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// ---- host-side dispatch of launch codes to template arguments -------------------------------
// The launchers call a generic lambda with a tag and recover the type as
// `typename decltype(tag)::type`, so each launch site is written once for every type.
template <typename T>
struct type_tag {
  using type = T;
};

// dtype code of activations, gradients and tables: 0 fp32, 1 bf16, 2 fp16
template <typename F>
void with_dtype(int code, F&& f) {
  if (code == 1) f(type_tag<__nv_bfloat16>{});
  else if (code == 2) f(type_tag<__half>{});
  else f(type_tag<float>{});
}

// one of two types by a flag (64- or 32-bit ids, 32- or 64-bit sort keys)
template <typename IfTrue, typename IfFalse, typename F>
void with_type_if(bool flag, F&& f) {
  if (flag) f(type_tag<IfTrue>{});
  else f(type_tag<IfFalse>{});
}

// ---- small fixed-size vectors of fp32 ---------------------------------------------------
template <int VEC>
struct FVec {
  float v[VEC];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = 0.f;
  }
  __device__ __forceinline__ void fma(float a, const FVec& x) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = fmaf(a, x.v[i], v[i]);
  }
  __device__ __forceinline__ void add(const FVec& x) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] += x.v[i];
  }
  __device__ __forceinline__ void scale(float a) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] *= a;
  }
};

// Read-only fp32 row fragment (tables are immutable during the forward kernel).
template <int VEC>
__device__ __forceinline__ FVec<VEC> ld_f32(const float* p) {
  FVec<VEC> r;
  if constexpr (VEC == 4) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = __ldg(p + i);
  }
  return r;
}

// Plain (coherent) fp32 load: used for read-modify-write of weights / optimizer state.
template <int VEC>
__device__ __forceinline__ FVec<VEC> ld_f32_rw(const float* p) {
  FVec<VEC> r;
  if constexpr (VEC == 8) {
    const float4 a = *reinterpret_cast<const float4*>(p);
    const float4 b = *reinterpret_cast<const float4*>(p + 4);
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  } else if constexpr (VEC == 4) {
    float4 t = *reinterpret_cast<const float4*>(p);
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = p[i];
  }
  return r;
}

template <int VEC>
__device__ __forceinline__ void st_f32(float* p, const FVec<VEC>& x) {
  if constexpr (VEC == 8) {
    *reinterpret_cast<float4*>(p) = make_float4(x.v[0], x.v[1], x.v[2], x.v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(x.v[4], x.v[5], x.v[6], x.v[7]);
  } else if constexpr (VEC == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(x.v[0], x.v[1], x.v[2], x.v[3]);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = x.v[i];
  }
}

// 16-bit activation types on the wire: bf16 (default mixed precision) and fp16 (the reference's
// `mixed_float16` policy, dist_model_parallel.py:866).
template <typename T>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  if constexpr (std::is_same<T, __half>::value) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  } else {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
  }
}
template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (std::is_same<T, __half>::value) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
template <typename T>
__device__ __forceinline__ float to_f32(T v) {
  if constexpr (std::is_same<T, float>::value) return v;
  else if constexpr (std::is_same<T, __half>::value) return __half2float(v);
  else return __bfloat162float(v);
}
template <typename T>
__device__ __forceinline__ T from_f32(float v) {
  if constexpr (std::is_same<T, float>::value) return v;
  else if constexpr (std::is_same<T, __half>::value) return __float2half_rn(v);
  else return __float2bfloat16_rn(v);
}

// Typed load of an activation / gradient fragment (fp32, bf16 or fp16 in memory -> fp32
// registers).  Plain loads: the source may be memory written by another GPU before a signal.
template <typename T, int VEC>
__device__ __forceinline__ FVec<VEC> ld_act(const T* p) {
  if constexpr (sizeof(T) == 4) {
    return ld_f32_rw<VEC>(reinterpret_cast<const float*>(p));
  } else if constexpr (VEC == 8) {
    FVec<VEC> r;
    const uint4 t = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack2<T>(w[i]);
      r.v[2 * i] = f.x;
      r.v[2 * i + 1] = f.y;
    }
    return r;
  } else if constexpr (VEC == 4) {
    FVec<VEC> r;
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    const float2 fa = unpack2<T>(t.x), fb = unpack2<T>(t.y);
    r.v[0] = fa.x; r.v[1] = fa.y; r.v[2] = fb.x; r.v[3] = fb.y;
    return r;
  } else {
    FVec<VEC> r;
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = to_f32<T>(p[i]);
    return r;
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void st_act(T* p, const FVec<VEC>& x) {
  if constexpr (sizeof(T) == 4) {
    st_f32<VEC>(reinterpret_cast<float*>(p), x);
  } else if constexpr (VEC == 8) {
    uint4 t;
    t.x = pack2<T>(x.v[0], x.v[1]);
    t.y = pack2<T>(x.v[2], x.v[3]);
    t.z = pack2<T>(x.v[4], x.v[5]);
    t.w = pack2<T>(x.v[6], x.v[7]);
    *reinterpret_cast<uint4*>(p) = t;
  } else if constexpr (VEC == 4) {
    uint2 t;
    t.x = pack2<T>(x.v[0], x.v[1]);
    t.y = pack2<T>(x.v[2], x.v[3]);
    *reinterpret_cast<uint2*>(p) = t;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = from_f32<T>(x.v[i]);
  }
}

// ---- embedding tables: fp32, bf16 or fp16 storage, fp32 arithmetic -------------------------
// Read-only row fragment of a table in the forward (tables are immutable during the lookup):
// fp32 rows as float4 / scalars, 16-bit rows as one 16-byte (VEC 8), 8-byte (VEC 4) or 2-byte
// load per lane, converted to fp32 in registers.
template <typename TabT, int VEC>
__device__ __forceinline__ FVec<VEC> ld_tab(const TabT* p) {
  if constexpr (sizeof(TabT) == 4) {
    return ld_f32<VEC>(reinterpret_cast<const float*>(p));
  } else {
    FVec<VEC> r;
    if constexpr (VEC == 8) {
      const uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
      const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack2<TabT>(w[i]);
        r.v[2 * i] = f.x;
        r.v[2 * i + 1] = f.y;
      }
    } else if constexpr (VEC == 4) {
      const uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
      const float2 fa = unpack2<TabT>(t.x), fb = unpack2<TabT>(t.y);
      r.v[0] = fa.x; r.v[1] = fa.y; r.v[2] = fb.x; r.v[3] = fb.y;
    } else {
      const unsigned short* q = reinterpret_cast<const unsigned short*>(p);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const unsigned short b = __ldg(q + i);
        r.v[i] = to_f32<TabT>(*reinterpret_cast<const TabT*>(&b));
      }
    }
    return r;
  }
}

// Stochastic rounding of fp32 to bf16 / fp16 (the write-back of half-precision tables).
// The rule, mirrored bit for bit by ops/stochastic_rounding.py:
//   lo, hi = the neighbouring representable values of x in the target type; lo == hi -> x.
//   u = (r >> 8) * 2^-24;  result = u * (hi - lo) < x - lo ? hi : lo
// with every fp32 operation exact, so E[result] = x.  NaN / inf and values beyond the finite
// range convert as round-to-nearest does.  r is a 32-bit hash of (optimizer step, row key,
// column, stream): the result does not depend on which thread stores the element, and the step
// counter is device resident, so CUDA-graph replays draw fresh bits.  The stream separates the
// stored quantities: 0 the weight, 1 state0 (Adagrad accumulator / Adam m), 2 state1 (Adam v);
// it is folded into the step seed (step + 0x9e3779b9 + stream * 0x632be5ab).
__device__ __forceinline__ uint32_t sr_mix(uint32_t h) {
  h ^= h >> 16;
  h *= 0x7feb352du;
  h ^= h >> 15;
  h *= 0x846ca68bu;
  h ^= h >> 16;
  return h;
}
constexpr uint32_t kStreamWeight = 0, kStreamState0 = 1, kStreamState1 = 2;
__device__ __forceinline__ uint32_t sr_row_seed(uint32_t step, int64_t key,
                                                uint32_t stream = kStreamWeight) {
  uint32_t h = sr_mix(step + 0x9e3779b9u + stream * 0x632be5abu);
  h = sr_mix(h ^ static_cast<uint32_t>(key));
  return sr_mix(h ^ static_cast<uint32_t>(static_cast<uint64_t>(key) >> 32));
}
__device__ __forceinline__ uint32_t sr_bits(uint32_t row_seed, int col) {
  return sr_mix(row_seed ^ static_cast<uint32_t>(col));
}

template <typename T>
__device__ __forceinline__ unsigned short round_stochastic(float x, uint32_t r) {
  static_assert(sizeof(T) == 2, "16-bit target");
  unsigned short rn;
  float max_finite;
  if constexpr (std::is_same<T, __half>::value) {
    rn = __half_as_ushort(__float2half_rn(x));
    max_finite = 65504.f;
  } else {
    rn = __bfloat16_as_ushort(__float2bfloat16_rn(x));
    max_finite = 0x1.fep+127f;  // 3.3895e38
  }
  auto value = [](unsigned short b) {
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(b));
    else return __bfloat162float(__ushort_as_bfloat16(b));
  };
  const float rn_f = value(rn);
  // representable, NaN, +-inf or beyond the finite range: round to nearest
  if (rn_f == x || !(fabsf(x) <= max_finite)) return rn;
  // the other neighbour: one step away from rn towards x in the ordered 16-bit encoding
  const int ord = (rn & 0x8000) ? -static_cast<int>(rn & 0x7fff) : static_cast<int>(rn);
  const bool up = rn_f < x;
  const int o2 = up ? ord + 1 : ord - 1;
  const unsigned short nb = o2 >= 0 ? static_cast<unsigned short>(o2)
                                    : static_cast<unsigned short>(0x8000 | (-o2));
  const float nb_f = value(nb);
  const float lo = up ? rn_f : nb_f, hi = up ? nb_f : rn_f;
  const float u = __fmul_rn(static_cast<float>(r >> 8), 5.9604644775390625e-8f);  // 2^-24
  const bool take_hi = __fmul_rn(u, __fsub_rn(hi, lo)) < __fsub_rn(x, lo);
  const unsigned short lo_b = up ? rn : nb, hi_b = up ? nb : rn;
  return take_hi ? hi_b : lo_b;
}

// Plain (coherent) row fragment of a table for read-modify-write in the update kernels.
template <typename TabT, int VEC>
__device__ __forceinline__ FVec<VEC> ld_tab_rw(const TabT* p) {
  return ld_act<TabT, VEC>(p);
}

// Write-back of an updated row fragment (weights and optimizer state): fp32 as is, 16-bit with
// stochastic rounding keyed by (step, row key, column, stream).
template <typename TabT, int VEC>
__device__ __forceinline__ void st_tab(TabT* p, const FVec<VEC>& x, uint32_t step, int64_t key,
                                       int col, uint32_t stream = kStreamWeight) {
  if constexpr (sizeof(TabT) == 4) {
    st_f32<VEC>(reinterpret_cast<float*>(p), x);
  } else {
    const uint32_t seed = sr_row_seed(step, key, stream);
    unsigned short b[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) b[i] = round_stochastic<TabT>(x.v[i], sr_bits(seed, col + i));
    if constexpr (VEC == 4) {
      uint2 t;
      t.x = static_cast<uint32_t>(b[0]) | (static_cast<uint32_t>(b[1]) << 16);
      t.y = static_cast<uint32_t>(b[2]) | (static_cast<uint32_t>(b[3]) << 16);
      *reinterpret_cast<uint2*>(p) = t;
    } else {
      unsigned short* q = reinterpret_cast<unsigned short*>(p);
#pragma unroll
      for (int i = 0; i < VEC; ++i) q[i] = b[i];
    }
  }
}

// Fire-and-forget vector reduction into global memory (REDG.E.ADD.F32x4 on sm_90a).
template <int VEC>
__device__ __forceinline__ void red_add_f32(float* p, const FVec<VEC>& x) {
  if constexpr (VEC == 8) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(x.v[0]),
                 "f"(x.v[1]), "f"(x.v[2]), "f"(x.v[3])
                 : "memory");
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4),
                 "f"(x.v[4]), "f"(x.v[5]), "f"(x.v[6]), "f"(x.v[7])
                 : "memory");
  } else if constexpr (VEC == 4) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(x.v[0]),
                 "f"(x.v[1]), "f"(x.v[2]), "f"(x.v[3])
                 : "memory");
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i)
      asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p + i), "f"(x.v[i]) : "memory");
  }
}

// ---- system-scope flag primitives (peer-mapped signal pads) -----------------------------
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Signal pad layout: [channel][kMaxPeers] uint32 epochs, slot j of rank r's pad is written by
// rank j only.
constexpr int kFlagChannels = 16;
__device__ __forceinline__ uint32_t* flag_slot(void* pad, int channel, int writer) {
  return reinterpret_cast<uint32_t*>(pad) + channel * kMaxPeers + writer;
}

// A peer did not show up in time: record who (host-mapped word, readable after the trap) and
// kill the context.  Continuing would consume stale ids / gradients and corrupt the tables;
// a trapped kernel surfaces as a CUDA error on the host at the next synchronisation, which is
// what a stalled Horovod collective does for the reference (abort, not garbage).
__device__ __forceinline__ void peer_timeout_trap(int* error_flag, int peer) {
  if (error_flag != nullptr) {
    atomicExch_system(error_flag, 1 + peer);
    __threadfence_system();
  }
  __trap();
}

// Bounded spin (watchdog): returns false on timeout instead of hanging the GPU.
__device__ __forceinline__ bool wait_flag_ge(const uint32_t* p, uint32_t epoch,
                                             unsigned long long timeout_cycles) {
  unsigned long long start = clock64();
  unsigned spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(p) - epoch) < 0) {
    if ((++spins & 0x3ff) == 0 && timeout_cycles && (clock64() - start) > timeout_cycles)
      return false;
    __nanosleep(20);
  }
  return true;
}

// ---- producer / consumer signalling folded into data kernels (see SyncArgs in de_b200.h) ----
// Head: every block waits (its first `world` threads poll the *local* signal pad) before the
// kernel touches data a peer produced.
__device__ __forceinline__ void sync_head(const SyncArgs& a) {
  if (a.state == nullptr || (a.wait_ch < 0 && a.wait_abs_ch < 0)) return;
  const int t = threadIdx.x;
  if (t < a.world) {
    if (a.wait_ch >= 0) {
      const uint32_t target = a.state[a.wait_ch] + 1;
      if (!wait_flag_ge(flag_slot(a.flags.p[a.rank], a.wait_ch, t), target, a.timeout))
        peer_timeout_trap(a.error_flag, t);
    }
    if (a.wait_abs_ch >= 0) {
      const uint32_t target = a.state[kSyncChannels + a.wait_abs_ch];
      if (!wait_flag_ge(flag_slot(a.flags.p[a.rank], a.wait_abs_ch, t), target, a.timeout))
        peer_timeout_trap(a.error_flag, t);
    }
  }
  __syncthreads();
}

// Tail: the last block to finish publishes the signal (after a system-scope fence that orders
// every block's peer stores before the flag) and advances the epochs.  All threads of every
// block must call it (it contains __syncthreads).
__device__ __forceinline__ void sync_tail(const SyncArgs& a) {
  if (a.state == nullptr || (a.wait_ch < 0 && a.signal_ch < 0)) return;
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t done = atomicAdd(&a.state[2 * kSyncChannels + a.counter_slot], 1u);
    s_last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  const int t = threadIdx.x;
  if (a.signal_ch >= 0) {
    const uint32_t epoch = a.state[kSyncChannels + a.signal_ch] + 1;
    if (t < a.world) {
      __threadfence_system();
      st_release_sys(flag_slot(a.flags.p[t], a.signal_ch, a.rank), epoch);
    }
    __syncthreads();
    if (t == 0) a.state[kSyncChannels + a.signal_ch] = epoch;
  }
  if (t == 0) {
    if (a.wait_ch >= 0) a.state[a.wait_ch] += 1;
    a.state[2 * kSyncChannels + a.counter_slot] = 0;
  }
}

}  // namespace de
