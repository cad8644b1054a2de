// Deduplicated sparse backward for sm_90a: (row key, item) pairs -> radix sort -> unique
// segments -> one lane group per unique row sums its gradient rows (pulled from peer-mapped
// gradient buffers when world_size > 1) and applies the optimizer update in place
// (SGD / Adagrad / row-wise Adagrad / lazy Adam / lazy row-wise Adam / FTRL-Proximal), or emits
// (unique_ids, unique_grad) for an external optimizer.  The unique count never leaves the device (the reference copies it to the
// host to size its output: cc/kernels/embedding_lookup_kernels.cu:663-670).
//
// Capability parity: OffsetToWeightsAndRowId + cub sort/unique + segment reduce
// (embedding_lookup_kernels.cu:358-367, 603-775) + TF's sparse optimizer apply kernels.
#include <cub/cub.cuh>

#include "common.cuh"

namespace de {

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 32;
constexpr int kUnroll = 4;

template <typename IdT>
__device__ __forceinline__ const IdT* sample_ids(const InputDesc& D, const PeerPtrs& src,
                                                 int64_t src_batch, int64_t g, int& n,
                                                 int64_t& first_item) {
  if (D.offsets != nullptr) {
    int64_t a = D.offsets[g], b = D.offsets[g + 1];
    n = static_cast<int>(b - a);
    first_item = D.item_off + a;
    return reinterpret_cast<const IdT*>(D.ids) + a;
  }
  n = D.hotness;
  first_item = D.item_off + g * D.hotness;
  if (D.ids != nullptr) return reinterpret_cast<const IdT*>(D.ids) + g * D.hotness;
  int64_t s = g / src_batch;
  int64_t i = g - s * src_batch;
  return reinterpret_cast<const IdT*>(src.p[s]) + D.ids_off + i * D.hotness;
}

// key = global row (table key_base + fused row), item = f * batch + g.  Out-of-range ids get the
// sentinel key (= total rows) and sort to the end; the sort only needs log2(total rows + 1) bits.
template <typename IdT, typename KeyT>
__global__ void __launch_bounds__(kThreads)
build_keys_kernel(const InputDesc* __restrict__ descs, const TableDesc* __restrict__ tables,
                  int n_tables, int n_inputs, int64_t batch, int64_t src_batch,
                  const __grid_constant__ PeerPtrs src, KeyT* __restrict__ keys,
                  uint32_t* __restrict__ items) {
  const int64_t tiles_per_input = (batch + kTile - 1) / kTile;
  const int64_t total = tiles_per_input * n_inputs;
  const int lane = threadIdx.x & 31;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * (kThreads / 32);
  // ids outside a table get the key one past the last row: they sort to the end
  const int64_t sentinel = tables[n_tables - 1].key_base + tables[n_tables - 1].rows;
  for (int64_t t = warp; t < total; t += n_warps) {
    const int f = static_cast<int>(t / tiles_per_input);
    const int64_t g = (t - f * tiles_per_input) * kTile + lane;
    if (g >= batch) continue;
    const InputDesc D = descs[f];
    const int64_t key_base = tables[D.local_table].key_base;
    int n;
    int64_t first;
    const IdT* p = sample_ids<IdT>(D, src, src_batch, g, n, first);
    const uint32_t item = static_cast<uint32_t>(static_cast<int64_t>(f) * batch + g);
    for (int h = 0; h < n; ++h) {
      const int64_t id = static_cast<int64_t>(p[h]) + D.id_shift;
      const bool ok = static_cast<uint64_t>(id) < static_cast<uint64_t>(D.sub_rows);
      keys[first + h] = static_cast<KeyT>(ok ? key_base + D.row_base + id : sentinel);
      items[first + h] = item;
    }
  }
}

struct HeadPred {
  const int64_t* keys;
  __device__ __forceinline__ bool operator()(const int64_t& k) const {
    return k == 0 || keys[k] != keys[k - 1];
  }
};

__global__ void finish_segments_kernel(int64_t* seg_start, const int64_t* n_unique, int64_t n) {
  if (threadIdx.x == 0 && blockIdx.x == 0) seg_start[*n_unique] = n;
}

// The row pass of the sorted update kernels, their template parameter kRow (a bit set).  A launch
// that needs none of the bits takes the kRow = 0 instantiation; the bits give the row-wise
// optimizers and FTRL instantiations of their own, so the others keep their code and registers.
constexpr int kRowDecay = 1;  // weight decay on: the row pass reads the weights (s * g + wd * w)
constexpr int kRowAdam = 2;   // row-wise Adam (kind kOptRowwiseAdam)
constexpr int kRowFtrl = 4;   // FTRL-Proximal (kind kOptFtrl): no row pass, its own apply_update
// decoupled (AdamW-style) weight decay: apply_update scales the weight by 1 - lr * weight_decay
// before the step, and the gradient, the state and the row pass never see the decay (the row pass
// reads no weights)
constexpr int kRowDecoupled = 8;
// momentum SGD (kind kOptMomentum): no row pass, its own apply_update
constexpr int kRowMomentum = 16;

// Adam bias corrections from a device-resident step count (the host scalars baked into a captured
// CUDA graph would freeze at their capture-time values).
template <int kRow = 0>
__device__ __forceinline__ void resolve_step(OptimizerArgs& opt) {
  if (opt.step_ptr != nullptr && ((kRow & kRowAdam) || opt.kind == kOptAdam)) {
    const float t = *opt.step_ptr;
    opt.bias1 = 1.f - powf(opt.beta1, t);
    opt.bias2 = 1.f - powf(opt.beta2, t);
  }
}

// The step that keys the stochastic rounding of 16-bit tables and 16-bit optimizer state: the
// same device-resident count (kernels with fp32 tables and fp32 state do not use it and never
// read it).  The count is an fp32 word that advances by 1.0 per step, exact up to 2^24 = 16.7 M
// steps; beyond that it stops changing and every later step would draw the same bits for a given
// (row, column), which biases the rounding.  Runs that long need an integer counter here.
template <typename TabT, typename StateT>
__device__ __forceinline__ uint32_t rounding_step(const OptimizerArgs& opt) {
  if constexpr (sizeof(TabT) == 2 || sizeof(StateT) == 2) {
    return opt.step_ptr != nullptr ? static_cast<uint32_t>(*opt.step_ptr) : 0u;
  } else {
    return 0u;
  }
}

// ------------------------------------------------------------------ per-row optimizer apply
// FTRL's P(n) = n^(-lr_power); the default lr_power = -0.5 takes the square root.
__device__ __forceinline__ float ftrl_pow(float n, float lr_power) {
  return lr_power == -0.5f ? sqrtf(n) : powf(n, -lr_power);
}

// The weight is read in its storage type (TabT: fp32, bf16 or fp16) and the Adagrad / Adam state
// in its own (StateT: fp32 or bf16), both widened to fp32; the optimizer runs in fp32, the weight
// update uses the unrounded new state, and 16-bit weights and state are written back with
// stochastic rounding (st_tab), each from its own random stream.  Every row has exactly one
// writer per step, so each element is rounded once.  Row-wise state (row-wise Adagrad's
// accumulator, row-wise Adam's v) is always fp32.
//
// FTRL-Proximal (TensorFlow's ApplyFtrlV2 with Keras's beta), g the decayed gradient:
//   n' = n + g^2,  sigma = (P(n') - P(n)) / lr,  z += g + 2 l2_shrinkage w - sigma w,
//   w = |z| > l1 ? (sign(z) l1 - z) / ((beta + P(n')) / lr + 2 l2) : 0,  n = n'.
// At lr = 0 the row, n and z keep their bits (sigma would divide by zero).
//
// Momentum SGD (torch.optim.SGD, dampening 0), g the decayed gradient, b the buffer (state0):
//   b = fmaf(momentum, b, g);  w = fmaf(-lr, b, w),
//   nesterov: w = fmaf(-lr, fmaf(momentum, b, g), w).
// At momentum 0 both give SGD's fmaf(-lr, g, w) bit for bit.
template <typename TabT, int VEC, typename StateT = float, int kRow = 0>
__device__ __forceinline__ void apply_update(const TableDesc& T, const OptimizerArgs& opt,
                                             int64_t row, int col, const FVec<VEC>& g,
                                             float row_sumsq_mean, uint32_t step) {
  TabT* w = reinterpret_cast<TabT*>(T.weight) + row * T.width + col;
  FVec<VEC> wv = ld_tab_rw<TabT, VEC>(w);
  FVec<VEC> gv = g;
  if constexpr ((kRow & kRowDecoupled) != 0) {
    // w = (1 - lr wd) w, then the kind's step from the undecayed g: torch.optim.AdamW's order.
    // fmaf and __fmul_rn fix the roundings (no contraction into the step's subtraction).
    const float keep = fmaf(-opt.lr, opt.weight_decay, 1.f);
#pragma unroll
    for (int i = 0; i < VEC; ++i) wv.v[i] = __fmul_rn(wv.v[i], keep);
  } else {
    if (opt.weight_decay != 0.f) gv.fma(opt.weight_decay, wv);
  }
  if constexpr ((kRow & kRowFtrl) != 0) {
    if (opt.lr == 0.f) return;
    StateT* n = reinterpret_cast<StateT*>(T.state0) + row * T.width + col;
    StateT* z = reinterpret_cast<StateT*>(T.state1) + row * T.width + col;
    FVec<VEC> nv = ld_tab_rw<StateT, VEC>(n), zv = ld_tab_rw<StateT, VEC>(z);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float n_new = fmaf(gv.v[i], gv.v[i], nv.v[i]);
      const float p_new = ftrl_pow(n_new, opt.lr_power);
      const float sigma = (p_new - ftrl_pow(nv.v[i], opt.lr_power)) / opt.lr;
      zv.v[i] += gv.v[i] + 2.f * opt.l2_shrinkage * wv.v[i] - sigma * wv.v[i];
      const float q = (opt.ftrl_beta + p_new) / opt.lr + 2.f * opt.l2;
      wv.v[i] = fabsf(zv.v[i]) > opt.l1 ? (copysignf(opt.l1, zv.v[i]) - zv.v[i]) / q : 0.f;
      nv.v[i] = n_new;
    }
    st_tab<StateT, VEC>(n, nv, step, T.key_base + row, col, kStreamState0);
    st_tab<StateT, VEC>(z, zv, step, T.key_base + row, col, kStreamState1);
  } else if constexpr ((kRow & kRowMomentum) != 0) {
    StateT* b = reinterpret_cast<StateT*>(T.state0) + row * T.width + col;
    FVec<VEC> bv = ld_tab_rw<StateT, VEC>(b);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      bv.v[i] = fmaf(opt.momentum, bv.v[i], gv.v[i]);
      const float u = opt.nesterov ? fmaf(opt.momentum, bv.v[i], gv.v[i]) : bv.v[i];
      wv.v[i] = fmaf(-opt.lr, u, wv.v[i]);
    }
    st_tab<StateT, VEC>(b, bv, step, T.key_base + row, col, kStreamState0);
  } else if constexpr ((kRow & kRowAdam) != 0) {
    // row-wise Adam: m element-wise; row_sumsq_mean carries the row's new v (the caller advanced
    // state1[row])
    StateT* m = reinterpret_cast<StateT*>(T.state0) + row * T.width + col;
    FVec<VEC> mv = ld_tab_rw<StateT, VEC>(m);
    const float denom = sqrtf(row_sumsq_mean / opt.bias2) + opt.eps;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      mv.v[i] = opt.beta1 * mv.v[i] + (1.f - opt.beta1) * gv.v[i];
      const float mh = mv.v[i] / opt.bias1;
      wv.v[i] -= opt.lr * mh / denom;
    }
    st_tab<StateT, VEC>(m, mv, step, T.key_base + row, col, kStreamState0);
  } else if (opt.kind == kOptSGD) {
    wv.fma(-opt.lr, gv);
  } else if (opt.kind == kOptAdagrad) {
    StateT* a = reinterpret_cast<StateT*>(T.state0) + row * T.width + col;
    FVec<VEC> av = ld_tab_rw<StateT, VEC>(a);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      av.v[i] = fmaf(gv.v[i], gv.v[i], av.v[i]);
      wv.v[i] -= opt.lr * gv.v[i] / (sqrtf(av.v[i]) + opt.eps);
    }
    st_tab<StateT, VEC>(a, av, step, T.key_base + row, col, kStreamState0);
  } else if (opt.kind == kOptRowwiseAdagrad) {
    // state0[row] was already advanced by the caller; row_sumsq_mean carries the new value
    const float denom = sqrtf(row_sumsq_mean) + opt.eps;
#pragma unroll
    for (int i = 0; i < VEC; ++i) wv.v[i] -= opt.lr * gv.v[i] / denom;
  } else if (opt.kind == kOptAdam) {
    StateT* m = reinterpret_cast<StateT*>(T.state0) + row * T.width + col;
    StateT* v = reinterpret_cast<StateT*>(T.state1) + row * T.width + col;
    FVec<VEC> mv = ld_tab_rw<StateT, VEC>(m), vv = ld_tab_rw<StateT, VEC>(v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      mv.v[i] = opt.beta1 * mv.v[i] + (1.f - opt.beta1) * gv.v[i];
      vv.v[i] = opt.beta2 * vv.v[i] + (1.f - opt.beta2) * gv.v[i] * gv.v[i];
      const float mh = mv.v[i] / opt.bias1;
      const float vh = vv.v[i] / opt.bias2;
      wv.v[i] -= opt.lr * mh / (sqrtf(vh) + opt.eps);
    }
    st_tab<StateT, VEC>(m, mv, step, T.key_base + row, col, kStreamState0);
    st_tab<StateT, VEC>(v, vv, step, T.key_base + row, col, kStreamState1);
  }
  st_tab<TabT, VEC>(w, wv, step, T.key_base + row, col);
}

// Sum of the gradient rows of one unique key restricted to this lane's columns.
template <typename GradT, int VEC>
__device__ __forceinline__ FVec<VEC> reduce_segment(const InputDesc* __restrict__ descs,
                                                    const uint32_t* __restrict__ items,
                                                    int64_t k0, int64_t k1, int64_t batch,
                                                    int64_t grad_batch, int64_t grad_stride,
                                                    const PeerPtrs& grad, int col) {
  FVec<VEC> acc;
  acc.zero();
  int64_t k = k0;
  for (; k + kUnroll <= k1; k += kUnroll) {
    FVec<VEC> x[kUnroll];
    float w[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint32_t item = items[k + u];
      const int f = static_cast<int>(item / batch);
      const int64_t g = item - static_cast<int64_t>(f) * batch;
      const InputDesc& D = descs[f];
      const int64_t d = g / grad_batch;
      const int64_t i = g - d * grad_batch;
      w[u] = 1.f;
      if (D.combiner == 1) {
        const int n = D.offsets ? static_cast<int>(D.offsets[g + 1] - D.offsets[g]) : D.hotness;
        w[u] = 1.f / static_cast<float>(n);
      }
      x[u] = ld_act<GradT, VEC>(reinterpret_cast<const GradT*>(grad.p[d]) + i * grad_stride +
                                D.dst_col + col);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) acc.fma(w[u], x[u]);
  }
  for (; k < k1; ++k) {
    const uint32_t item = items[k];
    const int f = static_cast<int>(item / batch);
    const int64_t g = item - static_cast<int64_t>(f) * batch;
    const InputDesc& D = descs[f];
    const int64_t d = g / grad_batch;
    const int64_t i = g - d * grad_batch;
    float w = 1.f;
    if (D.combiner == 1) {
      const int n = D.offsets ? static_cast<int>(D.offsets[g + 1] - D.offsets[g]) : D.hotness;
      w = 1.f / static_cast<float>(n);
    }
    acc.fma(w, ld_act<GradT, VEC>(reinterpret_cast<const GradT*>(grad.p[d]) + i * grad_stride +
                                  D.dst_col + col));
  }
  return acc;
}

// One lane group per unique row.  TabT is the table's storage type, StateT that of the Adagrad /
// Adam / row-wise Adam m state; with_update_types() below says which combinations a launch takes.
// Row-wise Adagrad and row-wise Adam first reduce the row mean of the squared gradient over the
// lane group (pass 1) into their fp32 word per row.  With weight decay (kRow & kRowDecay) that is
// the decayed gradient (s * g + weight_decay * w), the gradient apply_update applies, so pass 1
// reads the weights.
template <typename GradT, int VEC, typename TabT, typename StateT, int kRow>
__device__ __forceinline__ void segment_update_body(
    const InputDesc* __restrict__ descs, const TableDesc* __restrict__ tables, int n_tables,
    int lpr, int64_t batch, int64_t grad_batch, int64_t grad_stride, const PeerPtrs& grad,
    const int64_t* __restrict__ sorted_keys, const uint32_t* __restrict__ sorted_items,
    const int64_t* __restrict__ seg_start, const int64_t* __restrict__ n_unique_p,
    const OptimizerArgs& opt_in, int64_t* __restrict__ emit_keys, float* __restrict__ emit_rows,
    int emit_width) {
  OptimizerArgs opt = opt_in;
  if (opt.lr_ptr != nullptr) opt.lr = *opt.lr_ptr;
  resolve_step<kRow>(opt);
  const uint32_t sr_step = rounding_step<TabT, StateT>(opt);
  const int64_t n_unique = *n_unique_p;
  const int64_t sentinel = tables[n_tables - 1].key_base + tables[n_tables - 1].rows;
  const int lane = threadIdx.x & 31;
  const int rpw = 32 / lpr;
  const int sub = lane / lpr, li = lane - sub * lpr;
  const unsigned group_mask = (lpr == 32) ? 0xffffffffu : (((1u << lpr) - 1u) << (sub * lpr));
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * (kThreads / 32);

  for (int64_t u0 = warp * rpw; u0 < n_unique; u0 += n_warps * rpw) {
    const int64_t u = u0 + sub;
    const bool active = u < n_unique;
    int64_t key = sentinel, k0 = 0, k1 = 0;
    if (active) {
      k0 = seg_start[u];
      k1 = seg_start[u + 1];
      key = sorted_keys[k0];
    }
    const bool valid = active && key < sentinel;
    int m = 0;
    if (valid) {
      while (m + 1 < n_tables && tables[m + 1].key_base <= key) ++m;
    }
    const TableDesc T = tables[m];
    const int64_t row = key - T.key_base;
    const int W = T.width;
    const int nvec = (W + VEC - 1) / VEC;

    float row_state = 0.f;
    if (!(kRow & (kRowFtrl | kRowMomentum)) &&
        ((kRow & kRowAdam) || opt.kind == kOptRowwiseAdagrad)) {
      // pass 1: mean of squared (scaled) gradient over the whole row
      float ss = 0.f;
      if (valid) {
        for (int c0 = 0; c0 < nvec; c0 += lpr) {
          const int cv = c0 + li;
          if (cv < nvec) {
            FVec<VEC> g = reduce_segment<GradT, VEC>(descs, sorted_items, k0, k1, batch,
                                                     grad_batch, grad_stride, grad, cv * VEC);
            if constexpr ((kRow & kRowDecay) != 0) {
              // the same fp32 operations as apply_update, so the same values
              g.scale(opt.grad_scale);
              g.fma(opt.weight_decay,
                    ld_tab_rw<TabT, VEC>(reinterpret_cast<const TabT*>(T.weight) + row * W +
                                         cv * VEC));
#pragma unroll
              for (int i = 0; i < VEC; ++i) ss = fmaf(g.v[i], g.v[i], ss);
            } else {
#pragma unroll
              for (int i = 0; i < VEC; ++i) {
                const float x = g.v[i] * opt.grad_scale;
                ss = fmaf(x, x, ss);
              }
            }
          }
        }
      }
      for (int off = lpr >> 1; off > 0; off >>= 1) ss += __shfl_xor_sync(group_mask, ss, off);
      if (valid) {
        float* st = reinterpret_cast<float*>((kRow & kRowAdam) ? T.state1 : T.state0) + row;
        if constexpr ((kRow & kRowAdam) != 0)
          row_state = opt.beta2 * *st + (1.f - opt.beta2) * (ss / static_cast<float>(W));
        else
          row_state = *st + ss / static_cast<float>(W);
        if (li == 0) *st = row_state;
      }
      __syncwarp(group_mask);
    }
    if (!valid) {
      if (active && opt.kind == kOptEmit && li == 0) emit_keys[u] = sentinel;
      continue;
    }
    if (opt.kind == kOptEmit && li == 0) emit_keys[u] = key;
    for (int c0 = 0; c0 < nvec; c0 += lpr) {
      const int cv = c0 + li;
      if (cv >= nvec) continue;
      const int col = cv * VEC;
      FVec<VEC> g = reduce_segment<GradT, VEC>(descs, sorted_items, k0, k1, batch, grad_batch,
                                               grad_stride, grad, col);
      g.scale(opt.grad_scale);
      if (opt.kind == kOptEmit) {
        st_f32<VEC>(emit_rows + u * emit_width + col, g);
      } else {
        apply_update<TabT, VEC, StateT, kRow>(T, opt, row, col, g, row_state, sr_step);
      }
    }
  }
}

// The bodies of the three update kernels stay separate inlined functions: folded into the kernels,
// they get a different register allocation from ptxas.
template <typename GradT, int VEC, typename TabT, typename StateT, int kRow>
__global__ void __launch_bounds__(kThreads) segment_update_kernel(
    const InputDesc* __restrict__ descs, const TableDesc* __restrict__ tables, int n_tables,
    int lpr, int64_t batch, int64_t grad_batch, int64_t grad_stride,
    const __grid_constant__ PeerPtrs grad, const int64_t* __restrict__ sorted_keys,
    const uint32_t* __restrict__ sorted_items, const int64_t* __restrict__ seg_start,
    const int64_t* __restrict__ n_unique_p, const __grid_constant__ OptimizerArgs opt_in,
    int64_t* __restrict__ emit_keys, float* __restrict__ emit_rows, int emit_width) {
  segment_update_body<GradT, VEC, TabT, StateT, kRow>(
      descs, tables, n_tables, lpr, batch, grad_batch, grad_stride, grad, sorted_keys,
      sorted_items, seg_start, n_unique_p, opt_in, emit_keys, emit_rows, emit_width);
}

// ------------------------------------------------------------------ occurrence-balanced update
// Power-law ids put a large share of all look-ups on a handful of rows (alpha = 1.05: ~7 % on one
// row), so "one lane group per unique row" serialises.  Here the *sorted occurrence list* is cut
// into fixed chunks of kChunk positions; a lane group walks one chunk, summing runs of equal
// keys.  A run that is a whole segment is applied directly; a segment that crosses a chunk border
// is accumulated with vector RED into the scratch row of the chunk where it starts and applied by
// `finalize_crossing_kernel`.  Work per lane group is constant no matter how skewed the ids are.
constexpr int kChunk = 32;
constexpr int kBalUnroll = 8;  // gradient rows in flight per lane group

template <typename GradT>
__device__ __forceinline__ FVec<4> load_weighted_grad(const InputDesc* __restrict__ descs,
                                                      uint32_t item, int64_t batch,
                                                      int64_t grad_batch, int64_t grad_stride,
                                                      const PeerPtrs& grad, int col, float& w,
                                                      bool& ok) {
  const int f = static_cast<int>(item / batch);
  const int64_t g = item - static_cast<int64_t>(f) * batch;
  const InputDesc& D = descs[f];
  const int64_t d = g / grad_batch;
  const int64_t i = g - d * grad_batch;
  w = 1.f;
  if (D.combiner == 1) {
    const int n = D.offsets ? static_cast<int>(D.offsets[g + 1] - D.offsets[g]) : D.hotness;
    w = 1.f / static_cast<float>(n);
  }
  ok = col < D.width;
  FVec<4> x;
  x.zero();
  if (ok)
    x = ld_act<GradT, 4>(reinterpret_cast<const GradT*>(grad.p[d]) + i * grad_stride + D.dst_col +
                         col);
  return x;
}

// start position of the segment that contains sorted position `pos` (binary search, O(log u))
__device__ __forceinline__ int64_t segment_start_of(const int64_t* __restrict__ seg_start,
                                                    int64_t n_unique, int64_t pos) {
  int64_t lo = 0, hi = n_unique;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (seg_start[mid] <= pos) lo = mid;
    else hi = mid;
  }
  return seg_start[lo];
}

__device__ __forceinline__ int find_table(const TableDesc* __restrict__ tables, int n_tables,
                                          int64_t key) {
  int m = 0;
  while (m + 1 < n_tables && tables[m + 1].key_base <= key) ++m;
  return m;
}

// Apply the optimizer to one row given the complete (scaled) gradient fragment of this lane.
// kRow: the row pass of row-wise Adagrad / row-wise Adam, or FTRL / momentum (see
// segment_update_body).
template <typename TabT, typename StateT, int kRow = 0>
__device__ __forceinline__ void apply_row(const TableDesc& T, const OptimizerArgs& opt,
                                          int64_t row, int col, FVec<4> g, int lpr,
                                          unsigned group_mask, uint32_t step) {
  const bool col_ok = col < T.width;
  float row_state = 0.f;
  if (!(kRow & (kRowFtrl | kRowMomentum)) &&
      ((kRow & kRowAdam) || opt.kind == kOptRowwiseAdagrad)) {
    float ss = 0.f;
    if (col_ok) {
      if constexpr ((kRow & kRowDecay) != 0) {
        // the row word takes the gradient apply_update applies: g + weight_decay * w
        FVec<4> gd = g;
        gd.fma(opt.weight_decay,
               ld_tab_rw<TabT, 4>(reinterpret_cast<const TabT*>(T.weight) + row * T.width + col));
#pragma unroll
        for (int i = 0; i < 4; ++i) ss = fmaf(gd.v[i], gd.v[i], ss);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) ss = fmaf(g.v[i], g.v[i], ss);
      }
    }
    for (int off = lpr >> 1; off > 0; off >>= 1) ss += __shfl_xor_sync(group_mask, ss, off);
    float* st = reinterpret_cast<float*>((kRow & kRowAdam) ? T.state1 : T.state0) + row;
    if constexpr ((kRow & kRowAdam) != 0)
      row_state = opt.beta2 * *st + (1.f - opt.beta2) * (ss / static_cast<float>(T.width));
    else
      row_state = *st + ss / static_cast<float>(T.width);
    __syncwarp(group_mask);
    if (col == 0) *st = row_state;
  }
  if (col_ok) apply_update<TabT, 4, StateT, kRow>(T, opt, row, col, g, row_state, step);
}

template <typename GradT, typename TabT, typename StateT, int kRow>
__device__ __forceinline__ void balanced_update_body(
    const InputDesc* __restrict__ descs, const TableDesc* __restrict__ tables, int n_tables,
    int lpr, int64_t batch, int64_t grad_batch, int64_t grad_stride, const PeerPtrs& grad,
    const int64_t* __restrict__ sorted_keys, const uint32_t* __restrict__ sorted_items,
    int64_t n_items, const int64_t* __restrict__ seg_start, const int64_t* __restrict__ n_unique_p,
    const OptimizerArgs& opt_in, float* __restrict__ scratch, int scratch_width) {
  OptimizerArgs opt = opt_in;
  if (opt.lr_ptr != nullptr) opt.lr = *opt.lr_ptr;
  resolve_step<kRow>(opt);
  const uint32_t sr_step = rounding_step<TabT, StateT>(opt);
  const int64_t n_unique = *n_unique_p;
  const int64_t sentinel = tables[n_tables - 1].key_base + tables[n_tables - 1].rows;
  const int lane = threadIdx.x & 31;
  const int rpw = 32 / lpr;
  const int sub = lane / lpr, li = lane - sub * lpr;
  const int col = li * 4;
  const unsigned group_mask = (lpr == 32) ? 0xffffffffu : (((1u << lpr) - 1u) << (sub * lpr));
  const int64_t n_chunks = (n_items + kChunk - 1) / kChunk;
  const int64_t group = ((static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5) * rpw +
                        sub;
  const int64_t n_groups = static_cast<int64_t>(gridDim.x) * (kThreads / 32) * rpw;

  for (int64_t chunk = group; chunk < n_chunks; chunk += n_groups) {
    const int64_t k0 = chunk * kChunk;
    const int64_t k1 = min(n_items, k0 + kChunk);
    FVec<4> acc;
    acc.zero();
    int64_t run_key = sorted_keys[k0];
    int64_t run_start = k0;
    for (int64_t kb = k0; kb < k1; kb += kBalUnroll) {
      int64_t key[kBalUnroll];
      FVec<4> x[kBalUnroll];
      float w[kBalUnroll];
      bool ok[kBalUnroll];
#pragma unroll
      for (int u = 0; u < kBalUnroll; ++u) {
        const int64_t k = kb + u;
        key[u] = sentinel;
        ok[u] = false;
        w[u] = 0.f;
        x[u].zero();
        if (k < k1) {
          key[u] = sorted_keys[k];
          if (key[u] < sentinel)
            x[u] = load_weighted_grad<GradT>(descs, sorted_items[k], batch, grad_batch,
                                             grad_stride, grad, col, w[u], ok[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < kBalUnroll; ++u) {
        const int64_t k = kb + u;
        if (k >= k1) break;
        if (key[u] != run_key) {
          // flush the finished run [run_start, k)
          if (run_key < sentinel) {
            const bool start_done = run_start > k0 || k0 == 0 || sorted_keys[k0 - 1] != run_key;
            const int m = find_table(tables, n_tables, run_key);
            const TableDesc T = tables[m];
            FVec<4> g = acc;
            g.scale(opt.grad_scale);
            if (start_done) {
              apply_row<TabT, StateT, kRow>(T, opt, run_key - T.key_base, col, g, lpr, group_mask, sr_step);
            } else if (col < T.width) {
              // continues a segment that started in an earlier chunk: that chunk owns the slot
              const int64_t s = segment_start_of(seg_start, n_unique, k0);
              red_add_f32<4>(scratch + (s / kChunk) * scratch_width + col, g);
            }
          }
          acc.zero();
          run_key = key[u];
          run_start = k;
        }
        if (ok[u]) acc.fma(w[u], x[u]);
      }
    }
    // last run of the chunk
    if (run_key < sentinel) {
      const bool start_done = run_start > k0 || k0 == 0 || sorted_keys[k0 - 1] != run_key;
      const bool end_done = k1 == n_items || sorted_keys[k1] != run_key;
      const int m = find_table(tables, n_tables, run_key);
      const TableDesc T = tables[m];
      FVec<4> g = acc;
      g.scale(opt.grad_scale);
      if (start_done && end_done) {
        apply_row<TabT, StateT, kRow>(T, opt, run_key - T.key_base, col, g, lpr, group_mask, sr_step);
      } else if (col < T.width) {
        const int64_t s = start_done ? run_start : segment_start_of(seg_start, n_unique, k0);
        red_add_f32<4>(scratch + (s / kChunk) * scratch_width + col, g);
      }
    }
  }
}

template <typename GradT, typename TabT, typename StateT, int kRow>
__global__ void __launch_bounds__(kThreads) balanced_update_kernel(
    const InputDesc* __restrict__ descs, const TableDesc* __restrict__ tables, int n_tables,
    int lpr, int64_t batch, int64_t grad_batch, int64_t grad_stride,
    const __grid_constant__ PeerPtrs grad, const int64_t* __restrict__ sorted_keys,
    const uint32_t* __restrict__ sorted_items, int64_t n_items,
    const int64_t* __restrict__ seg_start, const int64_t* __restrict__ n_unique_p,
    const __grid_constant__ OptimizerArgs opt_in, float* __restrict__ scratch, int scratch_width) {
  balanced_update_body<GradT, TabT, StateT, kRow>(
      descs, tables, n_tables, lpr, batch, grad_batch, grad_stride, grad, sorted_keys,
      sorted_items, n_items, seg_start, n_unique_p, opt_in, scratch, scratch_width);
}

// One lane group per chunk: if a segment that crosses the chunk's end border starts in this chunk,
// its complete gradient sits in the chunk's scratch row: apply it, then clear the row.
template <typename TabT, typename StateT, int kRow>
__device__ __forceinline__ void finalize_crossing_body(
    const TableDesc* __restrict__ tables, int n_tables, int lpr,
    const int64_t* __restrict__ sorted_keys, int64_t n_items, const OptimizerArgs& opt_in,
    float* __restrict__ scratch, int scratch_width) {
  OptimizerArgs opt = opt_in;
  if (opt.lr_ptr != nullptr) opt.lr = *opt.lr_ptr;
  resolve_step<kRow>(opt);
  const uint32_t sr_step = rounding_step<TabT, StateT>(opt);
  const int64_t sentinel = tables[n_tables - 1].key_base + tables[n_tables - 1].rows;
  const int lane = threadIdx.x & 31;
  const int rpw = 32 / lpr;
  const int sub = lane / lpr, li = lane - sub * lpr;
  const int col = li * 4;
  const unsigned group_mask = (lpr == 32) ? 0xffffffffu : (((1u << lpr) - 1u) << (sub * lpr));
  const int64_t n_chunks = (n_items + kChunk - 1) / kChunk;
  const int64_t group = ((static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) >> 5) * rpw +
                        sub;
  const int64_t n_groups = static_cast<int64_t>(gridDim.x) * (kThreads / 32) * rpw;
  for (int64_t chunk = group; chunk < n_chunks; chunk += n_groups) {
    const int64_t k0 = chunk * kChunk;
    const int64_t last = min(n_items, k0 + kChunk) - 1;
    if (last + 1 >= n_items) continue;
    const int64_t key = sorted_keys[last];
    if (key >= sentinel || sorted_keys[last + 1] != key) continue;  // nothing crosses the border
    // the crossing segment belongs to this chunk only if it starts inside it
    if (sorted_keys[k0] == key && k0 > 0 && sorted_keys[k0 - 1] == key) continue;
    const int m = find_table(tables, n_tables, key);
    const TableDesc T = tables[m];
    float* sp = scratch + chunk * scratch_width + col;
    FVec<4> g;
    g.zero();
    if (col < T.width) {
      g = ld_f32_rw<4>(sp);
      FVec<4> z;
      z.zero();
      st_f32<4>(sp, z);
    }
    apply_row<TabT, StateT, kRow>(T, opt, key - T.key_base, col, g, lpr, group_mask, sr_step);
  }
}

template <typename TabT, typename StateT, int kRow>
__global__ void __launch_bounds__(kThreads)
finalize_crossing_kernel(const TableDesc* __restrict__ tables, int n_tables, int lpr,
                         const int64_t* __restrict__ sorted_keys, int64_t n_items,
                         const __grid_constant__ OptimizerArgs opt_in, float* __restrict__ scratch,
                         int scratch_width) {
  finalize_crossing_body<TabT, StateT, kRow>(tables, n_tables, lpr, sorted_keys, n_items,
                                                  opt_in, scratch, scratch_width);
}

int grid_cap(int64_t work_warps, int sm_count, int per_sm) {
  int64_t blocks = (work_warps + (kThreads / 32) - 1) / (kThreads / 32);
  int64_t cap = static_cast<int64_t>(sm_count) * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

// The instantiation a sorted update launch takes: calls f(type_tag<TabT>, type_tag<StateT>,
// kRow).  Only Adagrad, Adam, row-wise Adam and FTRL read element-wise state, so every other
// optimizer takes the fp32-state kernels; row-wise Adam (kRowAdam) and FTRL (kRowFtrl) have
// kernels of their own; only the row-wise optimizers with weight decay read the weights in their
// row pass (kRowDecay); decoupled decay of the stateful kinds takes kRowDecoupled (SGD's
// decoupled update is its L2 update, so it stays on the plain kernels); momentum (kRowMomentum,
// fp32 or bf16 b, plain or decoupled) has kernels of its own, so the kinds above keep theirs; the
// emit path never touches the table, so one fp32-table instantiation serves every storage type.
template <typename F>
void with_update_types(const OptimizerArgs& opt, int table_dtype, int state_dtype, F&& f) {
  using Plain = std::integral_constant<int, 0>;
  const bool decoupled = opt.weight_decay_mode == kWeightDecayDecoupled &&
                         opt.weight_decay != 0.f && opt.kind != kOptSGD &&
                         opt.kind != kOptEmit && opt.kind != kOptFtrl;
  with_dtype(opt.kind == kOptEmit ? 0 : table_dtype, [&](auto tab) {
    if (opt.kind == kOptMomentum) {
      with_type_if<__nv_bfloat16, float>(state_dtype == 1, [&](auto state) {
        if (decoupled)
          f(tab, state, std::integral_constant<int, kRowMomentum | kRowDecoupled>{});
        else
          f(tab, state, std::integral_constant<int, kRowMomentum>{});
      });
    } else if (decoupled) {
      // Adagrad / Adam with fp32 or bf16 state; row-wise Adagrad and row-wise Adam (fp32 or bf16
      // m) without a weight read in their row pass
      const bool half = state_dtype == 1 && opt.kind != kOptRowwiseAdagrad;
      with_type_if<__nv_bfloat16, float>(half, [&](auto state) {
        if (opt.kind == kOptRowwiseAdam)
          f(tab, state, std::integral_constant<int, kRowAdam | kRowDecoupled>{});
        else
          f(tab, state, std::integral_constant<int, kRowDecoupled>{});
      });
    } else if (opt.kind == kOptFtrl) {
      with_type_if<__nv_bfloat16, float>(state_dtype == 1, [&](auto state) {
        f(tab, state, std::integral_constant<int, kRowFtrl>{});
      });
    } else if (opt.kind == kOptRowwiseAdam) {
      with_type_if<__nv_bfloat16, float>(state_dtype == 1, [&](auto state) {
        if (opt.weight_decay != 0.f)
          f(tab, state, std::integral_constant<int, kRowAdam | kRowDecay>{});
        else
          f(tab, state, std::integral_constant<int, kRowAdam>{});
      });
    } else if (state_dtype == 1 && (opt.kind == kOptAdagrad || opt.kind == kOptAdam)) {
      f(tab, type_tag<__nv_bfloat16>{}, Plain{});
    } else if (opt.kind == kOptRowwiseAdagrad && opt.weight_decay != 0.f) {
      f(tab, type_tag<float>{}, std::integral_constant<int, kRowDecay>{});
    } else {
      f(tab, type_tag<float>{}, Plain{});
    }
  });
}

}  // namespace

void launch_build_keys(const InputDesc* descs, const TableDesc* tables, int n_tables, int n_inputs,
                       int64_t batch, int64_t src_batch, const PeerPtrs& src, bool ids64, void* keys,
                       uint32_t* items, int sm_count, cudaStream_t stream, bool keys32) {
  if (n_inputs <= 0 || batch <= 0) return;
  const int64_t tiles = ((batch + kTile - 1) / kTile) * n_inputs;
  const int grid = grid_cap(tiles, sm_count, 8);
  with_type_if<int64_t, int32_t>(ids64, [&](auto id) {
    using IdT = typename decltype(id)::type;
    with_type_if<uint32_t, int64_t>(keys32, [&](auto key) {
      using KeyT = typename decltype(key)::type;
      build_keys_kernel<IdT, KeyT><<<grid, kThreads, 0, stream>>>(
          descs, tables, n_tables, n_inputs, batch, src_batch, src, reinterpret_cast<KeyT*>(keys),
          items);
    });
  });
}

size_t sort_pairs_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, static_cast<const int64_t*>(nullptr),
                                  static_cast<int64_t*>(nullptr),
                                  static_cast<const uint32_t*>(nullptr),
                                  static_cast<uint32_t*>(nullptr), n, 0, 64);
  return bytes;
}

void sort_pairs(void* temp, size_t temp_bytes, const int64_t* keys_in, int64_t* keys_out,
                const uint32_t* items_in, uint32_t* items_out, int64_t n, int end_bit,
                cudaStream_t stream) {
  if (n <= 0) return;
  // keys are < total_rows + 1, callers pass end_bit = bit_length(total_rows)
  cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, items_in, items_out, n, 0,
                                  end_bit, stream);
}

size_t unique_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::CountingInputIterator<int64_t> it(0);
  HeadPred pred{nullptr};
  cub::DeviceSelect::If(nullptr, bytes, it, static_cast<int64_t*>(nullptr),
                        static_cast<int64_t*>(nullptr), n, pred);
  return bytes;
}

void unique_segments(void* temp, size_t temp_bytes, const int64_t* sorted_keys, int64_t n,
                     int64_t* seg_start, int64_t* n_unique, cudaStream_t stream) {
  if (n <= 0) {
    cudaMemsetAsync(n_unique, 0, sizeof(int64_t), stream);
    return;
  }
  cub::CountingInputIterator<int64_t> it(0);
  HeadPred pred{sorted_keys};
  cub::DeviceSelect::If(temp, temp_bytes, it, seg_start, n_unique, n, pred, stream);
  finish_segments_kernel<<<1, 32, 0, stream>>>(seg_start, n_unique, n);
}

void launch_segment_update(const InputDesc* descs, const TableDesc* tables, int n_tables,
                           int64_t batch, int64_t grad_batch, int64_t grad_stride,
                           const PeerPtrs& grad, const int64_t* sorted_keys,
                           const uint32_t* sorted_items, const int64_t* seg_start,
                           const int64_t* n_unique, int64_t n_items, const OptimizerArgs& opt,
                           int64_t* emit_keys, float* emit_rows, int max_width, int act_dtype,
                           bool vec4, int sm_count, cudaStream_t stream, int table_dtype,
                           int state_dtype) {
  const int emit_width = max_width;
  if (n_items <= 0 || n_tables <= 0) return;
  // lanes per row from the widest table of this launch (narrower tables leave lanes idle)
  const int vec = vec4 ? 4 : 1;
  const int lpr = [&] {
    int v = (emit_width + vec - 1) / vec;
    int p = 1;
    while (p < v && p < 32) p <<= 1;
    return p;
  }();
  const int rpw = 32 / lpr;
  const int64_t warps = (n_items + rpw - 1) / rpw;
  const int grid = grid_cap(warps, sm_count, 8);
  with_update_types(opt, table_dtype, state_dtype, [&](auto tab, auto state, auto row_pass) {
    using TabT = typename decltype(tab)::type;
    using StateT = typename decltype(state)::type;
    constexpr int kRow = decltype(row_pass)::value;
    with_dtype(act_dtype, [&](auto grad_t) {
      using GradT = typename decltype(grad_t)::type;
      auto launch = [&](auto kernel) {
        kernel<<<grid, kThreads, 0, stream>>>(descs, tables, n_tables, lpr, batch, grad_batch,
                                              grad_stride, grad, sorted_keys, sorted_items,
                                              seg_start, n_unique, opt, emit_keys, emit_rows,
                                              emit_width);
      };
      if (vec4) launch(segment_update_kernel<GradT, 4, TabT, StateT, kRow>);
      else launch(segment_update_kernel<GradT, 1, TabT, StateT, kRow>);
    });
  });
}

// Occurrence-balanced variant (vec4, tables up to 128 columns wide, fused optimizers only).
// `scratch` holds ceil(n_items / 32) rows of `scratch_width` floats and must be all zero on entry;
// it is all zero again on exit.
bool launch_balanced_update(const InputDesc* descs, const TableDesc* tables, int n_tables,
                            int64_t batch, int64_t grad_batch, int64_t grad_stride,
                            const PeerPtrs& grad, const int64_t* sorted_keys,
                            const uint32_t* sorted_items, int64_t n_items,
                            const int64_t* seg_start, const int64_t* n_unique,
                            const OptimizerArgs& opt, float* scratch, int scratch_width,
                            int max_width, int act_dtype, int sm_count, cudaStream_t stream,
                            int table_dtype, int state_dtype) {
  if (n_items <= 0 || n_tables <= 0) return true;
  if (max_width > 128 || max_width % 4 || scratch_width % 4 || opt.kind == kOptEmit) return false;
  int lpr = 1;
  while (lpr < max_width / 4 && lpr < 32) lpr <<= 1;
  const int rpw = 32 / lpr;
  const int64_t n_chunks = (n_items + kChunk - 1) / kChunk;
  const int grid = grid_cap((n_chunks + rpw - 1) / rpw, sm_count, 8);
  with_update_types(opt, table_dtype, state_dtype, [&](auto tab, auto state, auto row_pass) {
    using TabT = typename decltype(tab)::type;
    using StateT = typename decltype(state)::type;
    constexpr int kRow = decltype(row_pass)::value;
    with_dtype(act_dtype, [&](auto grad_t) {
      using GradT = typename decltype(grad_t)::type;
      balanced_update_kernel<GradT, TabT, StateT, kRow><<<grid, kThreads, 0, stream>>>(
          descs, tables, n_tables, lpr, batch, grad_batch, grad_stride, grad, sorted_keys,
          sorted_items, n_items, seg_start, n_unique, opt, scratch, scratch_width);
    });
    finalize_crossing_kernel<TabT, StateT, kRow><<<grid, kThreads, 0, stream>>>(
        tables, n_tables, lpr, sorted_keys, n_items, opt, scratch, scratch_width);
  });
  return cudaGetLastError() == cudaSuccess;
}

}  // namespace de
