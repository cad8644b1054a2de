// TORCH_LIBRARY registration of the native ops (namespace de_b200) and the symmetric-memory
// runtime (cudaMalloc + CUDA IPC peer mapping).  Compiled with the host compiler only; the
// kernels live in the .cu files behind the plain C++ launchers of de_b200.h.
//
// Capability parity: op schemas + OpKernel classes of the reference
// (cc/ops/embedding_lookup_ops.cc:24-101, cc/kernels/embedding_lookup_kernels.cc:28-187).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "de_b200.h"

namespace {

using at::Tensor;

#define DE_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    TORCH_CHECK(_e == cudaSuccess, "CUDA error in " #expr ": ", cudaGetErrorString(_e)); \
  } while (0)

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

int sm_count() {
  static int cached = -1;
  if (cached < 0) cached = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  return cached;
}

de::PeerPtrs to_peers(at::IntArrayRef ptrs) {
  TORCH_CHECK(ptrs.size() <= de::kMaxPeers, "at most ", de::kMaxPeers, " peers are supported");
  de::PeerPtrs p;
  std::memset(&p, 0, sizeof(p));
  for (size_t i = 0; i < ptrs.size(); ++i) p.p[i] = reinterpret_cast<void*>(ptrs[i]);
  return p;
}

void check_launch() {
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "kernel launch failed: ", cudaGetErrorString(e));
}

// ------------------------------------------------------------------ signalling contexts
// One per CommContext: the peer-mapped signal pads, this rank's epoch words and the watchdog.
// Ops take `int[] sync` = {handle, wait_ch, wait_abs_ch, signal_ch, counter_slot} (empty = none).
struct SyncCtx {
  de::PeerPtrs flags;
  uint32_t* state;
  int* error_flag;
  unsigned long long timeout;
  int rank, world;
};
std::vector<SyncCtx>& sync_ctxs() {
  static std::vector<SyncCtx> v;
  return v;
}
std::mutex& sync_mutex() {
  static std::mutex m;
  return m;
}

int64_t sync_ctx_create(at::IntArrayRef flag_ptrs, Tensor state, int64_t rank, int64_t world,
                        int64_t timeout_cycles, int64_t error_ptr) {
  TORCH_CHECK(state.is_cuda() && state.scalar_type() == at::kInt && state.is_contiguous() &&
                  state.numel() >= de::kSyncStateWords,
              "sync state must be an int32 CUDA tensor of >= ", de::kSyncStateWords, " words");
  SyncCtx c;
  c.flags = to_peers(flag_ptrs);
  c.state = reinterpret_cast<uint32_t*>(state.data_ptr<int>());
  c.error_flag = reinterpret_cast<int*>(error_ptr);
  c.timeout = static_cast<unsigned long long>(timeout_cycles);
  c.rank = static_cast<int>(rank);
  c.world = static_cast<int>(world);
  std::lock_guard<std::mutex> lock(sync_mutex());
  sync_ctxs().push_back(c);
  return static_cast<int64_t>(sync_ctxs().size()) - 1;
}

de::SyncArgs to_sync(at::IntArrayRef spec) {
  de::SyncArgs a = de::no_sync();
  if (spec.size() == 0) return a;
  TORCH_CHECK(spec.size() == 5, "sync spec = {handle, wait_ch, wait_abs_ch, signal_ch, slot}");
  SyncCtx c;
  {
    std::lock_guard<std::mutex> lock(sync_mutex());
    TORCH_CHECK(spec[0] >= 0 && spec[0] < static_cast<int64_t>(sync_ctxs().size()),
                "unknown sync context");
    c = sync_ctxs()[spec[0]];
  }
  for (int i = 1; i <= 3; ++i)
    TORCH_CHECK(spec[i] >= -1 && spec[i] < de::kSyncChannels, "sync channel out of range");
  TORCH_CHECK(spec[4] >= 0 && spec[4] < 2 * de::kSyncChannels, "sync counter slot out of range");
  a.flags = c.flags;
  a.state = c.state;
  a.error_flag = c.error_flag;
  a.timeout = c.timeout;
  a.rank = c.rank;
  a.world = c.world;
  a.wait_ch = static_cast<int32_t>(spec[1]);
  a.wait_abs_ch = static_cast<int32_t>(spec[2]);
  a.signal_ch = static_cast<int32_t>(spec[3]);
  a.counter_slot = static_cast<int32_t>(spec[4]);
  return a;
}

int dtype_code(at::ScalarType t) {
  if (t == at::kFloat) return 0;
  if (t == at::kBFloat16) return 1;
  if (t == at::kHalf) return 2;
  TORCH_CHECK(false, "activations / gradients must be fp32, bf16 or fp16");
  return -1;
}

void sync_only(at::IntArrayRef sync) {
  de::launch_sync_only(to_sync(sync), cur_stream());
  check_launch();
}

// ------------------------------------------------------------------ descriptor-driven ops
std::vector<int64_t> struct_sizes() {
  return {static_cast<int64_t>(sizeof(de::InputDesc)), static_cast<int64_t>(sizeof(de::TableDesc)),
          static_cast<int64_t>(de::kMaxPeers), static_cast<int64_t>(sizeof(de::GradRoute)),
          static_cast<int64_t>(de::kSyncStateWords),
          static_cast<int64_t>(sizeof(de::CacheRemap))};
}

void lookup_fwd(const Tensor& descs, int64_t n_inputs, int64_t batch, int64_t src_batch,
                int64_t dst_batch, int64_t dst_stride, at::IntArrayRef src_ptrs,
                at::IntArrayRef dst_ptrs, int64_t rot, bool ids64, int64_t act_dtype, bool vec4,
                at::IntArrayRef sync, int64_t tile_samples, int64_t table_dtype, bool vec8) {
  TORCH_CHECK(descs.is_cuda(), "descs must live on the GPU");
  TORCH_CHECK(table_dtype >= 0 && table_dtype <= 2, "table_dtype: 0 fp32, 1 bf16, 2 fp16");
  c10::cuda::CUDAGuard guard(descs.device());
  de::launch_lookup_fwd(reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
                        static_cast<int>(n_inputs), batch, src_batch, dst_batch, dst_stride,
                        to_peers(src_ptrs), to_peers(dst_ptrs), static_cast<int>(rot), ids64,
                        static_cast<int>(act_dtype), vec4, sm_count(), cur_stream(),
                        to_sync(sync), static_cast<int>(tile_samples),
                        static_cast<int>(table_dtype), vec8);
  check_launch();
}

void scatter_add_bwd(const Tensor& descs, int64_t n_inputs, int64_t batch, int64_t src_batch,
                     int64_t grad_batch, int64_t grad_stride, at::IntArrayRef src_ptrs,
                     at::IntArrayRef grad_ptrs, int64_t rot, double scale, int64_t scale_ptr,
                     bool ids64, int64_t act_dtype, bool vec4, bool vec8, at::IntArrayRef sync,
                     bool staged) {
  TORCH_CHECK(descs.is_cuda(), "descs must live on the GPU");
  c10::cuda::CUDAGuard guard(descs.device());
  de::launch_scatter_add_bwd(reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
                             static_cast<int>(n_inputs), batch, src_batch, grad_batch, grad_stride,
                             to_peers(src_ptrs), to_peers(grad_ptrs), static_cast<int>(rot),
                             static_cast<float>(scale), reinterpret_cast<const float*>(scale_ptr),
                             ids64, static_cast<int>(act_dtype), vec4, sm_count(), cur_stream(),
                             vec8, to_sync(sync), staged);
  check_launch();
}

int bit_length(int64_t v) {
  int b = 0;
  while (v > 0) {
    ++b;
    v >>= 1;
  }
  return b < 1 ? 1 : b;
}

// Build (row key, item) pairs for every looked-up id, sort by key, and find the unique rows.
// Returns (sorted_keys, sorted_items, seg_start, n_unique[1]); nothing is copied to the host.
// The first-party radix sort / head compaction (radix_sort.cu) is the default; DE_B200_SORT=cub
// routes the deduplicated update through the CUB calls of the CUDA toolkit instead (A/B only)
bool use_own_sort() {
  static const bool own = [] {
    const char* v = std::getenv("DE_B200_SORT");
    return !(v != nullptr && std::string(v) == "cub");
  }();
  return own;
}

// standalone entry points of the first-party sort / head compaction (tests, micro-benchmarks)
std::tuple<Tensor, Tensor> radix_sort_pairs(const Tensor& keys, const Tensor& items,
                                            int64_t end_bit) {
  TORCH_CHECK(keys.is_cuda() && keys.scalar_type() == at::kLong && keys.is_contiguous());
  TORCH_CHECK(items.is_cuda() && items.scalar_type() == at::kInt && items.is_contiguous() &&
              items.numel() == keys.numel());
  c10::cuda::CUDAGuard guard(keys.device());
  const int64_t n = keys.numel();
  TORCH_CHECK(n < (int64_t(1) << 31), "own radix sort: too many items");
  Tensor ka = keys.clone(), ia = items.clone();
  Tensor kb = at::empty_like(ka), ib = at::empty_like(ia);
  if (n == 0) return {ka, ia};
  Tensor temp = at::empty({static_cast<int64_t>(de::radix_sort_temp_bytes(n))},
                          at::TensorOptions().device(keys.device()).dtype(at::kByte));
  int where = de::radix_sort_pairs(temp.data_ptr(), ka.data_ptr<int64_t>(),
                                   reinterpret_cast<uint32_t*>(ia.data_ptr<int>()),
                                   kb.data_ptr<int64_t>(),
                                   reinterpret_cast<uint32_t*>(ib.data_ptr<int>()), n,
                                   static_cast<int>(end_bit), cur_stream());
  check_launch();
  if (where == 0) return {ka, ia};
  return {kb, ib};
}

// (int32 keys in [0, 2^32) read as unsigned, int32 items) -> (int64 sorted keys, sorted items)
std::tuple<Tensor, Tensor> radix_sort_pairs32(const Tensor& keys, const Tensor& items,
                                              int64_t end_bit) {
  TORCH_CHECK(keys.is_cuda() && keys.scalar_type() == at::kInt && keys.is_contiguous());
  TORCH_CHECK(items.is_cuda() && items.scalar_type() == at::kInt && items.is_contiguous() &&
              items.numel() == keys.numel());
  c10::cuda::CUDAGuard guard(keys.device());
  const int64_t n = keys.numel();
  TORCH_CHECK(n < (int64_t(1) << 31), "own radix sort: too many items");
  Tensor ka = keys.clone(), ia = items.clone();
  Tensor kb = at::empty_like(ka), ib = at::empty_like(ia);
  Tensor out = at::empty({n}, keys.options().dtype(at::kLong));
  if (n == 0) return {out, ia};
  Tensor temp = at::empty({static_cast<int64_t>(de::radix_sort_temp_bytes(n))},
                          at::TensorOptions().device(keys.device()).dtype(at::kByte));
  int where = de::radix_sort_pairs32(
      temp.data_ptr(), reinterpret_cast<uint32_t*>(ka.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(ia.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(kb.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(ib.data_ptr<int>()), out.data_ptr<int64_t>(), n,
      static_cast<int>(end_bit), cur_stream());
  check_launch();
  return {out, where == 0 ? ia : ib};
}

std::tuple<Tensor, Tensor> head_segments(const Tensor& sorted_keys) {
  TORCH_CHECK(sorted_keys.is_cuda() && sorted_keys.scalar_type() == at::kLong &&
              sorted_keys.is_contiguous());
  c10::cuda::CUDAGuard guard(sorted_keys.device());
  const int64_t n = sorted_keys.numel();
  auto i64 = at::TensorOptions().device(sorted_keys.device()).dtype(at::kLong);
  Tensor seg_start = at::empty({n + 1}, i64);
  Tensor n_unique = at::zeros({1}, i64);
  if (n == 0) return {seg_start, n_unique};
  Tensor temp = at::empty({static_cast<int64_t>(de::head_segments_temp_bytes(n))},
                          at::TensorOptions().device(sorted_keys.device()).dtype(at::kByte));
  de::head_segments(temp.data_ptr(), sorted_keys.data_ptr<int64_t>(), n,
                    seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), cur_stream());
  check_launch();
  return {seg_start, n_unique};
}

std::tuple<Tensor, Tensor, Tensor, Tensor> sort_items(const Tensor& descs, const Tensor& tables,
                                                      int64_t n_tables, int64_t n_inputs,
                                                      int64_t batch, int64_t src_batch,
                                                      at::IntArrayRef src_ptrs, bool ids64,
                                                      int64_t n_items, int64_t total_rows,
                                                      bool prefill_sentinel) {
  TORCH_CHECK(descs.is_cuda() && tables.is_cuda());
  // item = input * batch + sample is stored in 32 bits (sparse_update_kernels.cu)
  TORCH_CHECK(n_inputs * batch < (int64_t(1) << 32),
              "sorted update: n_inputs * batch = ", n_inputs * batch, " does not fit 32-bit items");
  c10::cuda::CUDAGuard guard(descs.device());
  auto stream = cur_stream();
  auto i64 = at::TensorOptions().device(descs.device()).dtype(at::kLong);
  auto i32 = at::TensorOptions().device(descs.device()).dtype(at::kInt);
  // ragged inputs reserve capacity: unused slots keep the sentinel key and sort to the end
  Tensor keys = prefill_sentinel ? at::full({n_items}, total_rows, i64) : at::empty({n_items}, i64);
  Tensor keys_sorted = at::empty({n_items}, i64);
  Tensor items = at::empty({n_items}, i32), items_sorted = at::empty({n_items}, i32);
  Tensor seg_start = at::empty({n_items + 1}, i64);
  Tensor n_unique = at::zeros({1}, i64);
  if (n_items == 0) return {keys_sorted, items_sorted, seg_start, n_unique};
  if (use_own_sort() && total_rows < (int64_t(1) << 32) - 1) {
    // every key (and the sentinel = total_rows) fits 32 bits: sort (uint32, uint32) pairs, the
    // last pass widens the keys for the update kernels
    TORCH_CHECK(n_items < (int64_t(1) << 31), "own radix sort: too many items");
    Tensor k32a = prefill_sentinel
                      ? at::full({n_items}, static_cast<int64_t>(static_cast<int32_t>(
                                                static_cast<uint32_t>(total_rows))), i32)
                      : at::empty({n_items}, i32);
    Tensor k32b = at::empty({n_items}, i32);
    de::launch_build_keys(reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
                          reinterpret_cast<const de::TableDesc*>(tables.data_ptr()),
                          static_cast<int>(n_tables), static_cast<int>(n_inputs), batch,
                          src_batch, to_peers(src_ptrs), ids64, k32a.data_ptr(),
                          reinterpret_cast<uint32_t*>(items.data_ptr<int>()), sm_count(), stream,
                          true);
    check_launch();
    size_t sort_bytes = de::radix_sort_temp_bytes(n_items);
    size_t head_bytes = de::head_segments_temp_bytes(n_items);
    Tensor temp = at::empty({static_cast<int64_t>(std::max(sort_bytes, head_bytes))},
                            at::TensorOptions().device(descs.device()).dtype(at::kByte));
    int where = de::radix_sort_pairs32(
        temp.data_ptr(), reinterpret_cast<uint32_t*>(k32a.data_ptr<int>()),
        reinterpret_cast<uint32_t*>(items.data_ptr<int>()),
        reinterpret_cast<uint32_t*>(k32b.data_ptr<int>()),
        reinterpret_cast<uint32_t*>(items_sorted.data_ptr<int>()),
        keys_sorted.data_ptr<int64_t>(), n_items, bit_length(total_rows), stream);
    if (where == 0) std::swap(items, items_sorted);
    de::head_segments(temp.data_ptr(), keys_sorted.data_ptr<int64_t>(), n_items,
                      seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), stream);
    check_launch();
    return {keys_sorted, items_sorted, seg_start, n_unique};
  }
  de::launch_build_keys(reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
                        reinterpret_cast<const de::TableDesc*>(tables.data_ptr()),
                        static_cast<int>(n_tables), static_cast<int>(n_inputs), batch, src_batch,
                        to_peers(src_ptrs), ids64, keys.data_ptr<int64_t>(),
                        reinterpret_cast<uint32_t*>(items.data_ptr<int>()), sm_count(), stream);
  check_launch();
  if (use_own_sort()) {
    TORCH_CHECK(n_items < (int64_t(1) << 31), "own radix sort: too many items");
    size_t sort_bytes = de::radix_sort_temp_bytes(n_items);
    size_t head_bytes = de::head_segments_temp_bytes(n_items);
    Tensor temp = at::empty({static_cast<int64_t>(std::max(sort_bytes, head_bytes))},
                            at::TensorOptions().device(descs.device()).dtype(at::kByte));
    int where = de::radix_sort_pairs(temp.data_ptr(), keys.data_ptr<int64_t>(),
                                     reinterpret_cast<uint32_t*>(items.data_ptr<int>()),
                                     keys_sorted.data_ptr<int64_t>(),
                                     reinterpret_cast<uint32_t*>(items_sorted.data_ptr<int>()),
                                     n_items, bit_length(total_rows), stream);
    if (where == 0) {
      std::swap(keys, keys_sorted);
      std::swap(items, items_sorted);
    }
    de::head_segments(temp.data_ptr(), keys_sorted.data_ptr<int64_t>(), n_items,
                      seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), stream);
    check_launch();
    return {keys_sorted, items_sorted, seg_start, n_unique};
  }
  size_t sort_bytes = de::sort_pairs_temp_bytes(n_items);
  size_t uniq_bytes = de::unique_temp_bytes(n_items);
  Tensor temp = at::empty({static_cast<int64_t>(std::max(sort_bytes, uniq_bytes)) + 16},
                          at::TensorOptions().device(descs.device()).dtype(at::kByte));
  de::sort_pairs(temp.data_ptr(), sort_bytes, keys.data_ptr<int64_t>(),
                 keys_sorted.data_ptr<int64_t>(),
                 reinterpret_cast<const uint32_t*>(items.data_ptr<int>()),
                 reinterpret_cast<uint32_t*>(items_sorted.data_ptr<int>()), n_items,
                 bit_length(total_rows), stream);
  de::unique_segments(temp.data_ptr(), uniq_bytes, keys_sorted.data_ptr<int64_t>(), n_items,
                      seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), stream);
  check_launch();
  return {keys_sorted, items_sorted, seg_start, n_unique};
}

void segment_update(const Tensor& descs, const Tensor& tables, int64_t n_tables, int64_t batch,
                    int64_t grad_batch, int64_t grad_stride, at::IntArrayRef grad_ptrs,
                    const Tensor& sorted_keys, const Tensor& sorted_items, const Tensor& seg_start,
                    const Tensor& n_unique, int64_t opt_kind, double lr, double eps, double beta1,
                    double beta2, double bias1, double bias2, double grad_scale,
                    double weight_decay, int64_t lr_ptr, const c10::optional<Tensor>& emit_keys,
                    const c10::optional<Tensor>& emit_rows, int64_t max_width, int64_t act_dtype,
                    bool vec4, const c10::optional<Tensor>& scratch, int64_t step_ptr,
                    int64_t table_dtype, int64_t state_dtype, double lr_power = -0.5,
                    double l1 = 0.0, double l2 = 0.0, double l2_shrinkage = 0.0,
                    double ftrl_beta = 0.0) {
  c10::cuda::CUDAGuard guard(descs.device());
  TORCH_CHECK(table_dtype >= 0 && table_dtype <= 2, "table_dtype: 0 fp32, 1 bf16, 2 fp16");
  TORCH_CHECK(state_dtype == 0 || state_dtype == 1, "state_dtype: 0 fp32, 1 bf16");
  de::OptimizerArgs opt;
  opt.kind = static_cast<int32_t>(opt_kind);
  opt.lr = static_cast<float>(lr);
  opt.eps = static_cast<float>(eps);
  opt.beta1 = static_cast<float>(beta1);
  opt.beta2 = static_cast<float>(beta2);
  opt.bias1 = static_cast<float>(bias1);
  opt.bias2 = static_cast<float>(bias2);
  opt.grad_scale = static_cast<float>(grad_scale);
  opt.weight_decay = static_cast<float>(weight_decay);
  opt.lr_ptr = reinterpret_cast<const float*>(lr_ptr);
  opt.step_ptr = reinterpret_cast<const float*>(step_ptr);
  opt.lr_power = static_cast<float>(lr_power);
  opt.l1 = static_cast<float>(l1);
  opt.l2 = static_cast<float>(l2);
  opt.l2_shrinkage = static_cast<float>(l2_shrinkage);
  opt.ftrl_beta = static_cast<float>(ftrl_beta);
  if (opt.kind == de::kOptEmit) TORCH_CHECK(emit_keys.has_value() && emit_rows.has_value());
  // occurrence-balanced path: immune to id skew (needs a zeroed scratch of >= n_items/32 rows)
  if (scratch.has_value() && vec4 && max_width <= 128 && opt.kind != de::kOptEmit) {
    const int64_t n_items = sorted_keys.numel();
    const int64_t sw = (max_width + 3) / 4 * 4;
    TORCH_CHECK(scratch->scalar_type() == at::kFloat && scratch->is_contiguous() &&
                    scratch->numel() >= ((n_items + 31) / 32) * sw,
                "scratch too small for the balanced update");
    bool ok = de::launch_balanced_update(
        reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
        reinterpret_cast<const de::TableDesc*>(tables.data_ptr()), static_cast<int>(n_tables),
        batch, grad_batch, grad_stride, to_peers(grad_ptrs), sorted_keys.data_ptr<int64_t>(),
        reinterpret_cast<const uint32_t*>(sorted_items.data_ptr<int>()), n_items,
        seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), opt,
        scratch->data_ptr<float>(), static_cast<int>(sw), static_cast<int>(max_width),
        static_cast<int>(act_dtype), sm_count(), cur_stream(), static_cast<int>(table_dtype),
        static_cast<int>(state_dtype));
    TORCH_CHECK(ok, "balanced update launch failed");
    check_launch();
    return;
  }
  de::launch_segment_update(
      reinterpret_cast<const de::InputDesc*>(descs.data_ptr()),
      reinterpret_cast<const de::TableDesc*>(tables.data_ptr()), static_cast<int>(n_tables), batch,
      grad_batch, grad_stride, to_peers(grad_ptrs), sorted_keys.data_ptr<int64_t>(),
      reinterpret_cast<const uint32_t*>(sorted_items.data_ptr<int>()),
      seg_start.data_ptr<int64_t>(), n_unique.data_ptr<int64_t>(), sorted_keys.numel(), opt,
      emit_keys.has_value() ? emit_keys->data_ptr<int64_t>() : nullptr,
      emit_rows.has_value() ? emit_rows->data_ptr<float>() : nullptr, static_cast<int>(max_width),
      static_cast<int>(act_dtype), vec4, sm_count(), cur_stream(), static_cast<int>(table_dtype),
      static_cast<int>(state_dtype));
  check_launch();
}

// ------------------------------------------------------------------ single-table convenience
// (used by the Embedding layer; builds a one-entry descriptor on the fly)
Tensor upload_bytes(const void* host, size_t bytes, const at::Device& dev) {
  Tensor t = at::empty({static_cast<int64_t>(bytes)},
                       at::TensorOptions().device(dev).dtype(at::kByte));
  DE_CUDA_CHECK(cudaMemcpyAsync(t.data_ptr(), host, bytes, cudaMemcpyHostToDevice, cur_stream()));
  return t;
}

de::InputDesc single_desc(const void* table, const Tensor& values,
                          const c10::optional<Tensor>& offsets, int64_t hotness, int64_t rows,
                          int64_t width, int64_t combiner) {
  de::InputDesc d;
  std::memset(&d, 0, sizeof(d));
  d.table = table;
  d.ids = values.data_ptr();
  d.offsets = offsets.has_value() ? offsets->data_ptr<int64_t>() : nullptr;
  d.sub_rows = rows;
  d.width = static_cast<int32_t>(width);
  d.hotness = offsets.has_value() ? 0 : static_cast<int32_t>(hotness);
  d.combiner = static_cast<int32_t>(combiner);
  return d;
}

void check_ids(const Tensor& values, const c10::optional<Tensor>& offsets) {
  TORCH_CHECK(values.is_cuda() && values.is_contiguous(), "ids must be a contiguous CUDA tensor");
  TORCH_CHECK(values.scalar_type() == at::kInt || values.scalar_type() == at::kLong,
              "ids must be int32 or int64");
  if (offsets.has_value())
    TORCH_CHECK(offsets->is_cuda() && offsets->scalar_type() == at::kLong &&
                    offsets->is_contiguous(),
                "row_splits must be a contiguous int64 CUDA tensor");
}

// out[b, :] = combine_{k in sample b} param[ids[k], :]   (pooled in fp32, stored in the table's
// dtype like nn.EmbeddingBag, or in bf16 with out_bf16)
Tensor embedding_lookup_fwd(const Tensor& param, const Tensor& values,
                            const c10::optional<Tensor>& offsets, int64_t hotness, int64_t batch,
                            int64_t combiner, bool out_bf16) {
  const auto pt = param.scalar_type();
  TORCH_CHECK(param.is_cuda() && param.dim() == 2 &&
                  (pt == at::kFloat || pt == at::kBFloat16 || pt == at::kHalf) &&
                  param.is_contiguous(),
              "param must be a contiguous fp32, bf16 or fp16 [rows, width] CUDA tensor");
  check_ids(values, offsets);
  c10::cuda::CUDAGuard guard(param.device());
  const int64_t width = param.size(1);
  const int tdt = dtype_code(pt);
  Tensor out = at::empty({batch, width}, param.options().dtype(out_bf16 ? at::kBFloat16 : pt));
  if (batch == 0) return out;
  de::InputDesc d = single_desc(param.data_ptr(), values, offsets, hotness, param.size(0), width,
                                combiner);
  Tensor dd = upload_bytes(&d, sizeof(d), param.device());
  de::PeerPtrs src, dst;
  std::memset(&src, 0, sizeof(src));
  std::memset(&dst, 0, sizeof(dst));
  dst.p[0] = out.data_ptr();
  // samples per warp tile: ~64 gathered rows per tile, but never fewer samples than one warp
  // instruction covers (32 / lanes-per-row) - long segments then spread over many warps
  const int64_t avg_hot = std::max<int64_t>(1, values.numel() / std::max<int64_t>(batch, 1));
  int64_t lanes_per_row = 1;
  while (lanes_per_row < (width + 3) / 4 && lanes_per_row < 32) lanes_per_row *= 2;
  const int64_t ts = std::max<int64_t>(32 / lanes_per_row, std::min<int64_t>(32, 64 / avg_hot));
  // vector loads need the table's base on their own width: a contiguous view at an odd element
  // offset takes the scalar path
  const uintptr_t base = reinterpret_cast<uintptr_t>(param.data_ptr());
  const bool vec4 = width % 4 == 0 && base % (4 * param.element_size()) == 0;
  de::launch_lookup_fwd(reinterpret_cast<const de::InputDesc*>(dd.data_ptr()), 1, batch, batch,
                        batch, width, src, dst, 0, values.scalar_type() == at::kLong,
                        out_bf16 ? 1 : tdt, vec4, sm_count(), cur_stream(), de::no_sync(),
                        static_cast<int>(std::max<int64_t>(1, ts)), tdt,
                        width % 8 == 0 && base % 16 == 0);
  check_launch();
  return out;
}

// dst[ids[k], :] += scale * w * grad[sample(k), :]    (atomic; dst may be a dense grad buffer)
void embedding_scatter_add(Tensor dst, const Tensor& values, const c10::optional<Tensor>& offsets,
                           int64_t hotness, int64_t batch, int64_t combiner, const Tensor& grad,
                           double scale) {
  TORCH_CHECK(dst.is_cuda() && dst.dim() == 2 && dst.scalar_type() == at::kFloat &&
              dst.is_contiguous());
  TORCH_CHECK(grad.is_cuda() && grad.dim() == 2 && grad.stride(1) == 1);
  check_ids(values, offsets);
  if (batch == 0) return;
  c10::cuda::CUDAGuard guard(dst.device());
  const int64_t width = dst.size(1);
  de::InputDesc d = single_desc(dst.data_ptr(), values, offsets, hotness, dst.size(0), width,
                                combiner);
  Tensor dd = upload_bytes(&d, sizeof(d), dst.device());
  de::PeerPtrs src, gp;
  std::memset(&src, 0, sizeof(src));
  std::memset(&gp, 0, sizeof(gp));
  gp.p[0] = grad.data_ptr();
  const int gdt = dtype_code(grad.scalar_type());
  const int64_t gstride = grad.stride(0);
  // 4-wide gradient loads and 4-wide reductions into dst: both bases on the 16-byte grid
  const bool vec4 = (width % 4 == 0) && (gstride % 4 == 0) &&
                    (reinterpret_cast<uintptr_t>(grad.data_ptr()) % 16 == 0) &&
                    (reinterpret_cast<uintptr_t>(dst.data_ptr()) % 16 == 0);
  de::launch_scatter_add_bwd(reinterpret_cast<const de::InputDesc*>(dd.data_ptr()), 1, batch,
                             batch, batch, gstride, src, gp, 0, static_cast<float>(scale), nullptr,
                             values.scalar_type() == at::kLong, gdt, vec4, sm_count(),
                             cur_stream(), false, de::no_sync());
  check_launch();
}

// Deduplicated sparse gradient: (unique_ids sorted ascending, summed gradient rows)
std::tuple<Tensor, Tensor> embedding_lookup_grad(const Tensor& values,
                                                 const c10::optional<Tensor>& offsets,
                                                 int64_t hotness, int64_t batch, int64_t combiner,
                                                 const Tensor& grad, int64_t num_rows) {
  TORCH_CHECK(grad.is_cuda() && grad.dim() == 2 && grad.stride(1) == 1);
  check_ids(values, offsets);
  c10::cuda::CUDAGuard guard(grad.device());
  const int64_t width = grad.size(1);
  const int64_t n_items = values.numel();
  auto f32 = grad.options().dtype(at::kFloat);
  auto i64 = grad.options().dtype(at::kLong);
  if (n_items == 0) return {at::empty({0}, i64), at::empty({0, width}, f32)};
  de::InputDesc d = single_desc(nullptr, values, offsets, hotness, num_rows, width, combiner);
  de::TableDesc t;
  std::memset(&t, 0, sizeof(t));
  t.rows = num_rows;
  t.width = static_cast<int32_t>(width);
  Tensor dd = upload_bytes(&d, sizeof(d), grad.device());
  Tensor td = upload_bytes(&t, sizeof(t), grad.device());
  auto sorted = sort_items(dd, td, 1, 1, batch, batch, {}, values.scalar_type() == at::kLong,
                           n_items, num_rows, false);
  Tensor emit_keys = at::empty({n_items}, i64);
  Tensor emit_rows = at::empty({n_items, width}, f32);
  const int gdt = dtype_code(grad.scalar_type());
  const int64_t gstride = grad.stride(0);
  const bool vec4 = (width % 4 == 0) && (gstride % 4 == 0) &&
                    (reinterpret_cast<uintptr_t>(grad.data_ptr()) % 16 == 0);
  std::vector<int64_t> gp = {reinterpret_cast<int64_t>(grad.data_ptr())};
  segment_update(dd, td, 1, batch, batch, gstride, gp, std::get<0>(sorted), std::get<1>(sorted),
                 std::get<2>(sorted), std::get<3>(sorted), de::kOptEmit, 0, 0, 0, 0, 1, 1, 1.0, 0, 0,
                 emit_keys, emit_rows, width, gdt, vec4, c10::nullopt, 0, 0, 0);
  // sizing the IndexedSlices-style result needs the unique count on the host (compat path only)
  int64_t n_unique = std::get<3>(sorted).item<int64_t>();
  if (n_unique > 0) {
    // ids outside the table collapse into one trailing sentinel segment: drop it
    int64_t last = emit_keys.narrow(0, n_unique - 1, 1).item<int64_t>();
    if (last >= num_rows) --n_unique;
  }
  return {emit_keys.narrow(0, 0, n_unique), emit_rows.narrow(0, 0, n_unique)};
}

Tensor row_to_split(const Tensor& indices, int64_t num_rows) {
  TORCH_CHECK(indices.is_cuda() && indices.dim() == 2 && indices.size(1) == 2 &&
                  indices.scalar_type() == at::kLong && indices.is_contiguous(),
              "indices must be a contiguous int64 [nnz, 2] CUDA tensor");
  c10::cuda::CUDAGuard guard(indices.device());
  Tensor splits = at::empty({num_rows + 1}, indices.options());
  de::launch_row_to_split(indices.data_ptr<int64_t>(), indices.size(0), num_rows,
                          splits.data_ptr<int64_t>(), cur_stream());
  check_launch();
  return splits;
}

void hash_init(Tensor table) {
  TORCH_CHECK(table.is_cuda() && table.scalar_type() == at::kLong && table.is_contiguous());
  c10::cuda::CUDAGuard guard(table.device());
  de::launch_hash_init(table.data_ptr<int64_t>(), table.numel() / 2, cur_stream());
  check_launch();
}

Tensor integer_lookup(Tensor table, Tensor count, Tensor next_index, const Tensor& keys,
                      int64_t capacity) {
  TORCH_CHECK(table.is_cuda() && count.is_cuda() && next_index.is_cuda() && keys.is_cuda());
  TORCH_CHECK(table.scalar_type() == at::kLong && keys.scalar_type() == at::kLong &&
              next_index.scalar_type() == at::kLong && count.scalar_type() == at::kInt);
  c10::cuda::CUDAGuard guard(table.device());
  Tensor k = keys.contiguous();
  Tensor out = at::empty_like(k);
  de::launch_integer_lookup(table.data_ptr<int64_t>(), table.numel() / 2,
                            reinterpret_cast<uint32_t*>(count.data_ptr<int>()),
                            next_index.data_ptr<int64_t>(), k.data_ptr<int64_t>(), k.numel(),
                            capacity, out.data_ptr<int64_t>(), cur_stream());
  check_launch();
  return out;
}

// ------------------------------------------------------------------ communication ops
void barrier(at::IntArrayRef flag_ptrs, Tensor epoch, int64_t rank, int64_t world, int64_t channel,
             int64_t timeout_cycles, int64_t error_ptr) {
  c10::cuda::CUDAGuard guard(epoch.device());
  de::launch_barrier(to_peers(flag_ptrs), reinterpret_cast<uint32_t*>(epoch.data_ptr<int>()),
                     static_cast<int>(rank), static_cast<int>(world), static_cast<int>(channel),
                     static_cast<unsigned long long>(timeout_cycles),
                     reinterpret_cast<int*>(error_ptr), cur_stream());
  check_launch();
}

void allreduce(at::IntArrayRef buf_ptrs, at::IntArrayRef flag_ptrs, Tensor epoch, int64_t rank,
               int64_t world, int64_t n_elems, double scale, bool bf16, int64_t channel,
               int64_t timeout_cycles, int64_t error_ptr, int64_t mc_ptr, int64_t max_blocks) {
  c10::cuda::CUDAGuard guard(epoch.device());
  if (mc_ptr != 0) {
    de::launch_allreduce_multimem(reinterpret_cast<void*>(mc_ptr), to_peers(flag_ptrs),
                                  reinterpret_cast<uint32_t*>(epoch.data_ptr<int>()),
                                  static_cast<int>(rank), static_cast<int>(world), n_elems,
                                  static_cast<float>(scale), bf16, static_cast<int>(channel),
                                  static_cast<unsigned long long>(timeout_cycles),
                                  reinterpret_cast<int*>(error_ptr), sm_count(), cur_stream(),
                         static_cast<int>(max_blocks));
  } else {
    de::launch_allreduce(to_peers(buf_ptrs), to_peers(flag_ptrs),
                         reinterpret_cast<uint32_t*>(epoch.data_ptr<int>()),
                         static_cast<int>(rank), static_cast<int>(world), n_elems,
                         static_cast<float>(scale), bf16, static_cast<int>(channel),
                         static_cast<unsigned long long>(timeout_cycles),
                         reinterpret_cast<int*>(error_ptr), sm_count(), cur_stream(),
                         static_cast<int>(max_blocks));
  }
  check_launch();
}

void p2p_store_bench(const Tensor& src, int64_t dst_ptr, int64_t n_rows, int64_t row_bytes,
                     int64_t vec_bytes, int64_t dst_stride, int64_t unroll, int64_t blocks,
                     int64_t threads) {
  TORCH_CHECK(src.is_cuda() && src.is_contiguous() &&
              src.numel() * src.element_size() >= n_rows * row_bytes);
  TORCH_CHECK(row_bytes % vec_bytes == 0 && (vec_bytes == 4 || vec_bytes == 8 || vec_bytes == 16));
  TORCH_CHECK((row_bytes / vec_bytes >= 32 && (row_bytes / vec_bytes) % 32 == 0) ||
              32 % (row_bytes / vec_bytes) == 0);
  TORCH_CHECK(unroll >= 1 && unroll <= 8 && threads % 32 == 0 && threads <= 1024);
  c10::cuda::CUDAGuard guard(src.device());
  de::launch_p2p_store_bench(src.data_ptr(), reinterpret_cast<void*>(dst_ptr), n_rows,
                             static_cast<int>(row_bytes), static_cast<int>(vec_bytes), dst_stride,
                             static_cast<int>(unroll), static_cast<int>(blocks),
                             static_cast<int>(threads), cur_stream());
  check_launch();
}

// segs[j] = {dst_rank, src_elem_off, dst_elem_off, n_elems}: push id segments to their owners
void push_segments(const Tensor& segs, const Tensor& src, at::IntArrayRef dst_ptrs,
                   int64_t max_seg_elems, at::IntArrayRef sync) {
  TORCH_CHECK(segs.is_cuda() && segs.scalar_type() == at::kLong && segs.is_contiguous() &&
              segs.dim() == 2 && segs.size(1) == 4);
  TORCH_CHECK(src.is_cuda() && src.is_contiguous() &&
              (src.element_size() == 4 || src.element_size() == 8));
  c10::cuda::CUDAGuard guard(src.device());
  de::launch_push_segments(segs.data_ptr<int64_t>(), static_cast<int>(segs.size(0)),
                           src.data_ptr(), to_peers(dst_ptrs),
                           static_cast<int>(src.element_size()), max_seg_elems, sm_count(),
                           cur_stream(), to_sync(sync));
  check_launch();
}

// routes: raw bytes of a GradRoute array; src: local gradient rows [rows, *] (unit inner stride)
void push_grad(const Tensor& routes, int64_t n_routes, const Tensor& src, int64_t dst_dtype,
               double scale, at::IntArrayRef sync) {
  TORCH_CHECK(routes.is_cuda() && routes.scalar_type() == at::kByte &&
              routes.numel() >= n_routes * static_cast<int64_t>(sizeof(de::GradRoute)));
  TORCH_CHECK(src.is_cuda() && src.dim() == 2 && src.stride(1) == 1);
  c10::cuda::CUDAGuard guard(src.device());
  de::launch_push_grad(reinterpret_cast<const de::GradRoute*>(routes.data_ptr()),
                       static_cast<int>(n_routes), src.data_ptr(), src.stride(0),
                       dtype_code(src.scalar_type()), static_cast<int>(dst_dtype), src.size(0),
                       static_cast<float>(scale), sm_count(), cur_stream(), to_sync(sync));
  check_launch();
}

// Streamed push of an owner-major staging buffer (see de_b200.h PushPlan): src / dst pointers and
// bytes per row for every peer; counters[c] = rows of chunk c the producer has completed.
void stream_push(at::IntArrayRef src_ptrs, at::IntArrayRef dst_ptrs, at::IntArrayRef row_bytes,
                 const Tensor& counters, int64_t chunk_rows, int64_t rows, int64_t blocks,
                 at::IntArrayRef sync) {
  TORCH_CHECK(src_ptrs.size() == dst_ptrs.size() && src_ptrs.size() == row_bytes.size() &&
              src_ptrs.size() <= de::kMaxPeers);
  TORCH_CHECK(counters.is_cuda() && counters.scalar_type() == at::kInt && chunk_rows > 0 &&
              counters.numel() >= (rows + chunk_rows - 1) / chunk_rows);
  de::PushPlan plan;
  std::memset(&plan, 0, sizeof(plan));
  plan.n = static_cast<int32_t>(src_ptrs.size());
  for (size_t i = 0; i < src_ptrs.size(); ++i) {
    TORCH_CHECK(row_bytes[i] % 16 == 0 && src_ptrs[i] % 16 == 0 && dst_ptrs[i] % 16 == 0,
                "streamed push needs 16-byte aligned rows");
    plan.src[i] = reinterpret_cast<const void*>(src_ptrs[i]);
    plan.dst[i] = reinterpret_cast<void*>(dst_ptrs[i]);
    plan.row_bytes[i] = row_bytes[i];
  }
  c10::cuda::CUDAGuard guard(counters.device());
  de::SyncArgs sa = to_sync(sync);
  de::launch_stream_push(plan, reinterpret_cast<const uint32_t*>(counters.data_ptr<int>()),
                         static_cast<int>(chunk_rows), rows, sa.timeout, sa.error_flag,
                         static_cast<int>(blocks), cur_stream(), sa);
  check_launch();
}

// out[i, dst_col + c] = sum_s partial[s, i, src_col + c]; cols = int32 [n, 3] {src, dst, width}
void rowslice_reduce(const Tensor& partial, int64_t out_ptr, int64_t out_stride,
                     int64_t out_dtype, const Tensor& cols) {
  TORCH_CHECK(partial.is_cuda() && partial.dim() == 3 && partial.scalar_type() == at::kFloat &&
              partial.is_contiguous());
  TORCH_CHECK(cols.is_cuda() && cols.scalar_type() == at::kInt && cols.is_contiguous() &&
              cols.dim() == 2 && cols.size(1) == 3);
  c10::cuda::CUDAGuard guard(partial.device());
  de::launch_rowslice_reduce(partial.data_ptr<float>(), static_cast<int>(partial.size(0)),
                             partial.size(1), partial.size(2), reinterpret_cast<void*>(out_ptr),
                             out_stride, static_cast<int>(out_dtype), cols.data_ptr<int>(),
                             static_cast<int>(cols.size(0)), cur_stream());
  check_launch();
}

void gather_segments(const Tensor& segs, at::IntArrayRef src_ptrs, Tensor dst,
                     int64_t max_seg_elems) {
  TORCH_CHECK(segs.is_cuda() && segs.scalar_type() == at::kLong && segs.is_contiguous());
  TORCH_CHECK(dst.is_cuda() && dst.is_contiguous());
  c10::cuda::CUDAGuard guard(dst.device());
  de::launch_gather_segments(segs.data_ptr<int64_t>(), static_cast<int>(segs.size(0)),
                             to_peers(src_ptrs), dst.data_ptr(),
                             static_cast<int>(dst.element_size()), max_seg_elems, cur_stream());
  check_launch();
}

void gather_ragged(const Tensor& segs, at::IntArrayRef val_ptrs, at::IntArrayRef split_ptrs,
                   Tensor dst_vals, Tensor goff, int64_t b, int64_t max_cap) {
  TORCH_CHECK(segs.is_cuda() && segs.scalar_type() == at::kLong && segs.is_contiguous());
  TORCH_CHECK(goff.is_cuda() && goff.scalar_type() == at::kLong && dst_vals.is_cuda());
  c10::cuda::CUDAGuard guard(dst_vals.device());
  de::launch_gather_ragged(segs.data_ptr<int64_t>(), static_cast<int>(segs.size(0)),
                           to_peers(val_ptrs), to_peers(split_ptrs), dst_vals.data_ptr(),
                           goff.data_ptr<int64_t>(), b, static_cast<int>(val_ptrs.size()),
                           static_cast<int>(dst_vals.element_size()), max_cap, cur_stream());
  check_launch();
}

// dst[k] <- (slot ? src1[k] : src0[k]); the slot is read on the device (graph replay friendly)
void select_copy(at::TensorList src0, at::TensorList src1, at::TensorList dst,
                 const Tensor& slot_flag) {
  TORCH_CHECK(src0.size() == dst.size() && src1.size() == dst.size() && dst.size() <= 4);
  TORCH_CHECK(slot_flag.is_cuda() && slot_flag.scalar_type() == at::kInt);
  const void* s0[4];
  const void* s1[4];
  void* d[4];
  int64_t nb[4];
  for (size_t i = 0; i < dst.size(); ++i) {
    TORCH_CHECK(src0[i].is_contiguous() && src1[i].is_contiguous() && dst[i].is_contiguous());
    nb[i] = dst[i].numel() * dst[i].element_size();
    TORCH_CHECK(src0[i].numel() * src0[i].element_size() == nb[i] &&
                src1[i].numel() * src1[i].element_size() == nb[i] && nb[i] % 16 == 0,
                "select_copy segments must match and be multiples of 16 bytes");
    s0[i] = src0[i].data_ptr();
    s1[i] = src1[i].data_ptr();
    d[i] = dst[i].data_ptr();
  }
  c10::cuda::CUDAGuard guard(slot_flag.device());
  de::launch_select_copy(s0, s1, d, nb, static_cast<int>(dst.size()), slot_flag.data_ptr<int>(),
                         sm_count(), cur_stream());
  check_launch();
}

void copy_cast_2d(const Tensor& src, int64_t dst_ptr, int64_t dst_stride, int64_t dst_dtype,
                  double scale) {
  TORCH_CHECK(src.is_cuda() && src.dim() == 2 && src.stride(1) == 1);
  c10::cuda::CUDAGuard guard(src.device());
  de::launch_copy_cast_2d(src.data_ptr(), src.stride(0), reinterpret_cast<void*>(dst_ptr),
                          dst_stride, src.size(0), src.size(1), dtype_code(src.scalar_type()),
                          static_cast<int>(dst_dtype), static_cast<float>(scale), cur_stream());
  check_launch();
}

// ------------------------------------------------------------------ dense-side ops
void check_bf16_2d(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.dim() == 2 && t.scalar_type() == at::kBFloat16 && t.stride(1) == 1,
              name, " must be a 2-D bf16 CUDA tensor with unit inner stride");
}

// rows that start on `bytes`-byte boundaries (the interaction kernels stage feature rows with
// 16-byte cp.async and store gradient pairs as 4-byte words).  Messages carry strings only: with
// torch 2.11 an integer formatted into a TORCH_CHECK message crashes the process (SIGSEGV).
void check_row_alignment(const Tensor& t, int64_t bytes, const char* name) {
  TORCH_CHECK((t.stride(0) * 2) % bytes == 0 &&
                  reinterpret_cast<uintptr_t>(t.data_ptr()) % static_cast<uintptr_t>(bytes) == 0,
              name, bytes == 16 ? " rows must start on 16-byte boundaries"
                                : " rows must start on 4-byte boundaries");
}

// z[s] = [strict lower triangle of F F^T | bottom | zero pad], F = [bottom ; emb_0 ; ...]
void interact_fwd(const Tensor& bottom, const Tensor& emb, int64_t n_emb, Tensor z,
                  at::IntArrayRef sync) {
  check_bf16_2d(bottom, "bottom");
  check_bf16_2d(emb, "emb");
  check_bf16_2d(z, "z");
  c10::cuda::CUDAGuard guard(bottom.device());
  const int64_t dim = bottom.size(1);
  TORCH_CHECK(emb.size(1) == n_emb * dim, "emb must be [batch, n_emb * dim]");
  TORCH_CHECK(emb.size(0) >= bottom.size(0) && z.size(0) >= bottom.size(0),
              "emb and z need a row per row of bottom");
  check_row_alignment(bottom, 16, "bottom");
  check_row_alignment(emb, 16, "emb");
  const int64_t need = (n_emb + 1) * n_emb / 2 + dim;
  TORCH_CHECK(z.size(1) >= need, "z is too narrow");
  bool ok = de::launch_interact_fwd(bottom.data_ptr(), bottom.stride(0), emb.data_ptr(),
                                    emb.stride(0), static_cast<int>(n_emb), static_cast<int>(dim),
                                    z.data_ptr(), z.stride(0), static_cast<int>(z.size(1)),
                                    bottom.size(0), sm_count(), cur_stream(), to_sync(sync));
  TORCH_CHECK(ok, "unsupported interaction shape (n_emb <= 31, dim in {16,32,64,128})");
  check_launch();
}

void interact_bwd(const Tensor& bottom, const Tensor& emb, int64_t n_emb, const Tensor& dz,
                  Tensor dbottom, int64_t demb_ptr, int64_t demb_stride, double emb_grad_scale,
                  const c10::optional<Tensor>& routes, int64_t n_routes, at::IntArrayRef sync,
                  const c10::optional<Tensor>& done_counters, int64_t chunk_rows,
                  const c10::optional<Tensor>& apply_descs, double apply_scale,
                  int64_t apply_scale_ptr, bool apply_ids64) {
  // apply_descs: host uint8 tensor of n_emb InputDesc records, one per embedding row of F; a
  // record with a null table leaves that row to the routes, any other is updated in the kernel
  de::InteractApply apply{};
  if (apply_descs.has_value()) {
    const Tensor& a = *apply_descs;
    TORCH_CHECK(!a.is_cuda() && a.scalar_type() == at::kByte && a.is_contiguous(),
                "apply_descs must be a contiguous uint8 CPU tensor of InputDesc records");
    TORCH_CHECK(a.numel() == n_emb * static_cast<int64_t>(sizeof(de::InputDesc)),
                "apply_descs needs one InputDesc per embedding row");
    TORCH_CHECK(n_emb <= de::kMaxInteractApply, "apply_descs: at most 31 embedding rows");
    TORCH_CHECK(apply_scale_ptr % 4 == 0, "apply_scale_ptr must be 4-byte aligned");
    TORCH_CHECK(!done_counters.has_value(), "apply_descs cannot be combined with done_counters");
    const auto* d = reinterpret_cast<const de::InputDesc*>(a.data_ptr());
    for (int64_t f = 0; f < n_emb; ++f) {
      if (d[f].table == nullptr) continue;
      TORCH_CHECK(d[f].width == 128 && bottom.size(1) == 128,
                  "apply_descs: applied tables must be 128 wide, like the interaction");
      TORCH_CHECK(d[f].hotness == 1 && d[f].offsets == nullptr && d[f].ids != nullptr,
                  "apply_descs: applied inputs must be one-hot with direct ids");
      TORCH_CHECK(reinterpret_cast<uintptr_t>(d[f].table) % 16 == 0,
                  "apply_descs: tables must be 16-byte aligned");
      TORCH_CHECK(reinterpret_cast<uintptr_t>(d[f].ids) % (apply_ids64 ? 8 : 4) == 0,
                  "apply_descs: ids must be aligned to their element size");
      TORCH_CHECK(d[f].row_base >= 0 && d[f].sub_rows >= 0,
                  "apply_descs: row_base and sub_rows must not be negative");
      apply.table[f] = static_cast<float*>(const_cast<void*>(d[f].table));
      apply.ids[f] = d[f].ids;
      apply.row_base[f] = d[f].row_base;
      apply.sub_rows[f] = d[f].sub_rows;
      apply.id_shift[f] = d[f].id_shift;
      apply.mask |= 1u << f;
    }
    apply.scale = static_cast<float>(apply_scale);
    apply.scale_ptr = reinterpret_cast<const float*>(apply_scale_ptr);
    apply.ids64 = apply_ids64 ? 1 : 0;
  }
  check_bf16_2d(bottom, "bottom");
  check_bf16_2d(emb, "emb");
  check_bf16_2d(dz, "dz");
  check_bf16_2d(dbottom, "dbottom");
  if (routes.has_value()) {
    TORCH_CHECK(routes->is_cuda() && routes->scalar_type() == at::kByte &&
                routes->numel() >= n_routes * static_cast<int64_t>(sizeof(de::GradRoute)));
  } else {
    TORCH_CHECK(demb_ptr != 0, "interact_bwd needs an embedding-gradient buffer or routes");
  }
  const int64_t dim = bottom.size(1);
  const int64_t batch = bottom.size(0);
  TORCH_CHECK(emb.size(1) == n_emb * dim, "emb must be [batch, n_emb * dim]");
  TORCH_CHECK((n_emb + 1) * n_emb / 2 + dim <= dz.size(1), "dz is too narrow");
  TORCH_CHECK(dbottom.size(1) == dim, "dbottom must be [batch, dim]");
  TORCH_CHECK(emb.size(0) >= batch && dz.size(0) >= batch && dbottom.size(0) >= batch,
              "emb, dz and dbottom need a row per row of bottom");
  check_row_alignment(bottom, 16, "bottom");
  check_row_alignment(emb, 16, "emb");
  check_row_alignment(dbottom, 4, "dbottom");
  if (!routes.has_value())
    TORCH_CHECK(demb_stride % 2 == 0 && demb_ptr % 4 == 0,
                "embedding-gradient rows must start on 4-byte boundaries");
  if (done_counters.has_value()) {
    TORCH_CHECK(done_counters->is_cuda() && done_counters->scalar_type() == at::kInt &&
                    done_counters->is_contiguous(),
                "done_counters must be a contiguous int32 CUDA tensor");
    TORCH_CHECK(chunk_rows > 0, "chunk_rows must be positive with done_counters");
    TORCH_CHECK(done_counters->numel() >= (batch + chunk_rows - 1) / chunk_rows,
                "done_counters needs one counter per chunk of chunk_rows samples");
  }
  c10::cuda::CUDAGuard guard(bottom.device());
  bool ok = de::launch_interact_bwd(bottom.data_ptr(), bottom.stride(0), emb.data_ptr(),
                                    emb.stride(0), static_cast<int>(n_emb), static_cast<int>(dim),
                                    dz.data_ptr(), dz.stride(0), dbottom.data_ptr(),
                                    dbottom.stride(0), reinterpret_cast<void*>(demb_ptr),
                                    demb_stride, static_cast<float>(emb_grad_scale),
                                    bottom.size(0), sm_count(), cur_stream(),
                                    routes.has_value()
                                        ? reinterpret_cast<const de::GradRoute*>(routes->data_ptr())
                                        : nullptr,
                                    static_cast<int>(n_routes), to_sync(sync),
                                    done_counters.has_value()
                                        ? reinterpret_cast<uint32_t*>(done_counters->data_ptr<int>())
                                        : nullptr,
                                    static_cast<int>(chunk_rows),
                                    apply.mask != 0 ? &apply : nullptr);
  TORCH_CHECK(ok, "unsupported interaction shape (n_emb <= 31, dim in {32,64,128}; routed / "
                  "signalling launches need dim in {64,128} and 16-byte aligned rows)");
  check_launch();
}

// out[:, :out_len] = avg_pool1d(x[:, :n], stride) with "same" padding (bf16, unit inner strides)
void avgpool_fwd(const Tensor& x, int64_t n, Tensor out, int64_t stride) {
  check_bf16_2d(x, "x");
  check_bf16_2d(out, "out");
  const int64_t out_len = (n + stride - 1) / stride;
  TORCH_CHECK(x.size(1) >= n && out.size(1) >= out_len && out.size(0) == x.size(0));
  const int64_t pad = std::max<int64_t>(0, (out_len - 1) * stride + stride - n);
  c10::cuda::CUDAGuard guard(x.device());
  de::launch_avgpool_fwd(x.data_ptr(), x.stride(0), static_cast<int>(n), out.data_ptr(),
                         out.stride(0), static_cast<int>(out_len), static_cast<int>(stride),
                         static_cast<int>(pad / 2), x.size(0), cur_stream());
  check_launch();
}

// dx[:, :n] = gradient of avgpool_fwd for dout[:, :out_len]
void avgpool_bwd(const Tensor& dout, Tensor dx, int64_t n, int64_t stride) {
  check_bf16_2d(dout, "dout");
  check_bf16_2d(dx, "dx");
  const int64_t out_len = (n + stride - 1) / stride;
  TORCH_CHECK(dx.size(1) >= n && dout.size(1) >= out_len && dout.size(0) == dx.size(0));
  const int64_t pad = std::max<int64_t>(0, (out_len - 1) * stride + stride - n);
  c10::cuda::CUDAGuard guard(dx.device());
  de::launch_avgpool_bwd(dout.data_ptr(), dout.stride(0), static_cast<int>(out_len),
                         dx.data_ptr(), dx.stride(0), static_cast<int>(n),
                         static_cast<int>(stride), static_cast<int>(pad / 2), dx.size(0),
                         cur_stream());
  check_launch();
}

void relu_bwd_bias(Tensor dy, const Tensor& y, Tensor db) {
  check_bf16_2d(dy, "dy");
  check_bf16_2d(y, "y");
  TORCH_CHECK(dy.is_contiguous() && y.is_contiguous() && dy.size(1) % 8 == 0);
  TORCH_CHECK(y.sizes() == dy.sizes(), "y must have the shape of dy");
  // one thread per 8 columns in a 256-thread block
  TORCH_CHECK(dy.size(1) >= 8 && dy.size(1) <= 2048, "relu_bwd_bias supports 8..2048 columns");
  TORCH_CHECK(db.is_cuda() && db.scalar_type() == at::kFloat && db.numel() >= dy.size(1));
  c10::cuda::CUDAGuard guard(dy.device());
  de::launch_relu_bwd_bias(dy.data_ptr(), y.data_ptr(), db.data_ptr<float>(), dy.size(0),
                           static_cast<int>(dy.size(1)), cur_stream());
  check_launch();
}

// Host checks of the cross-network ops: a contiguous 2-D bf16 tensor on the device of `ref`,
// 16-byte aligned, with `cols` columns (a multiple of 8) and the rows of `ref`.  Messages carry
// strings only.
void check_cross(const Tensor& t, const Tensor& ref, int64_t cols, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.device() == ref.device(), name, " must be on the device of x0");
  TORCH_CHECK(t.dim() == 2 && t.scalar_type() == at::kBFloat16, name, " must be a 2-D bf16 tensor");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
  TORCH_CHECK(t.size(0) == ref.size(0) && t.size(1) == cols, name, " has the wrong shape");
  TORCH_CHECK(cols % 8 == 0 && cols > 0, name, " must have a positive multiple of 8 columns");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0, name,
              " must be 16-byte aligned");
}

// out = x0 * s + xl
void cross_fwd(const Tensor& x0, const Tensor& s, const Tensor& xl, Tensor out) {
  TORCH_CHECK(x0.dim() == 2, "x0 must be a 2-D bf16 tensor");
  const int64_t d = x0.size(1);
  check_cross(x0, x0, d, "x0");
  check_cross(s, x0, d, "s");
  check_cross(xl, x0, d, "xl");
  check_cross(out, x0, d, "out");
  c10::cuda::CUDAGuard guard(x0.device());
  de::launch_cross_fwd(x0.data_ptr(), s.data_ptr(), xl.data_ptr(), out.data_ptr(), x0.numel(),
                       sm_count(), cur_stream());
  check_launch();
}

// g = dy * x0 ; db += column sums of dy * x0 (fp32)
void cross_bwd(const Tensor& dy, const Tensor& x0, Tensor g, Tensor db) {
  TORCH_CHECK(x0.dim() == 2, "x0 must be a 2-D bf16 tensor");
  const int64_t d = x0.size(1);
  check_cross(x0, x0, d, "x0");
  check_cross(dy, x0, d, "dy");
  check_cross(g, x0, d, "g");
  TORCH_CHECK(db.device() == x0.device() && db.scalar_type() == at::kFloat && db.is_contiguous(),
              "db must be a contiguous fp32 tensor on the device of x0");
  TORCH_CHECK(db.numel() == d, "db must hold one element per column");
  c10::cuda::CUDAGuard guard(x0.device());
  de::launch_cross_bwd(dy.data_ptr(), x0.data_ptr(), g.data_ptr(), db.data_ptr<float>(),
                       x0.size(0), static_cast<int>(d), cur_stream());
  check_launch();
}

// d_chain + sum_l dy[l] * s[l]: the first D - B columns into dx0, the last B into d_bottom [rows, B]
void cross_dx0(const Tensor& d_chain, at::TensorList dy, at::TensorList s, Tensor dx0,
               Tensor d_bottom) {
  TORCH_CHECK(d_chain.dim() == 2, "d_chain must be a 2-D bf16 tensor");
  const int64_t d = d_chain.size(1);
  check_cross(d_chain, d_chain, d, "d_chain");
  check_cross(dx0, d_chain, d, "dx0");
  TORCH_CHECK(dy.size() == s.size(), "dy and s must have the same length");
  TORCH_CHECK(!dy.empty() && dy.size() <= static_cast<size_t>(de::kMaxCrossLayers),
              "cross_dx0 takes 1 to 8 layers");
  TORCH_CHECK(d_bottom.dim() == 2 && d_bottom.size(1) <= d,
              "d_bottom must be 2-D with at most the columns of d_chain");
  check_cross(d_bottom, d_chain, d_bottom.size(1), "d_bottom");
  de::CrossTerms terms{};
  for (size_t l = 0; l < dy.size(); ++l) {
    check_cross(dy[l], d_chain, d, "dy");
    check_cross(s[l], d_chain, d, "s");
    terms.dy[l] = dy[l].data_ptr();
    terms.s[l] = s[l].data_ptr();
  }
  terms.n = static_cast<int>(dy.size());
  c10::cuda::CUDAGuard guard(d_chain.device());
  de::launch_cross_dx0(d_chain.data_ptr(), terms, dx0.data_ptr(), d_bottom.data_ptr(),
                       d_chain.size(0), static_cast<int>(d),
                       static_cast<int>(d - d_bottom.size(1)), cur_stream());
  check_launch();
}

void head_loss(const Tensor& x, const Tensor& w, const Tensor& bias, const Tensor& labels,
               double inv_batch, Tensor dx, Tensor dw, Tensor db, Tensor dbias_prev,
               Tensor loss_sum, const c10::optional<Tensor>& logits) {
  check_bf16_2d(x, "x");
  TORCH_CHECK(x.is_contiguous() && dx.is_contiguous());
  TORCH_CHECK(w.scalar_type() == at::kBFloat16 && bias.scalar_type() == at::kBFloat16);
  TORCH_CHECK(labels.scalar_type() == at::kFloat && labels.is_contiguous());
  const int64_t batch = x.size(0), k = x.size(1);
  auto f32 = [](const Tensor& t, int64_t n, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous() &&
                    t.numel() >= n,
                name, " must be a contiguous fp32 CUDA tensor with enough elements");
  };
  TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.numel() == k, "w must hold K elements");
  TORCH_CHECK(bias.is_cuda() && bias.numel() >= 1, "bias must hold one element");
  TORCH_CHECK(labels.is_cuda() && labels.numel() == batch, "labels must hold one value per row");
  TORCH_CHECK(dx.is_cuda() && dx.scalar_type() == at::kBFloat16 && dx.sizes() == x.sizes(),
              "dx must be a bf16 tensor of the shape of x");
  f32(dw, k, "dw");
  f32(db, 1, "db");
  f32(dbias_prev, k, "dbias_prev");
  f32(loss_sum, 1, "loss_sum");
  if (logits.has_value()) f32(*logits, batch, "logits");
  c10::cuda::CUDAGuard guard(x.device());
  bool ok = de::launch_head_loss(x.data_ptr(), static_cast<int>(x.size(1)), w.data_ptr(),
                                 bias.data_ptr(), labels.data_ptr<float>(), x.size(0),
                                 static_cast<float>(inv_batch), dx.data_ptr(),
                                 dw.data_ptr<float>(), db.data_ptr<float>(),
                                 dbias_prev.data_ptr<float>(), loss_sum.data_ptr<float>(),
                                 logits.has_value() ? logits->data_ptr<float>() : nullptr,
                                 sm_count(), cur_stream());
  TORCH_CHECK(ok, "head_loss supports K in {64,128,256,512,1024}");
  check_launch();
}

// Evaluation head: probs = sigmoid(<x, w> + b); rows below *n_valid accumulate (+=) into the
// BinnedAUC histogram, the fp64 loss sum and the sample count.
void head_eval(const Tensor& x, const Tensor& w, const Tensor& bias, const Tensor& labels,
               const Tensor& n_valid, Tensor probs, Tensor hist, Tensor loss_sum, Tensor count) {
  check_bf16_2d(x, "x");
  TORCH_CHECK(x.is_contiguous(), "x must be contiguous");
  const int64_t batch = x.size(0), k = x.size(1);
  TORCH_CHECK(k == 64 || k == 128 || k == 256 || k == 512 || k == 1024,
              "head_eval supports K in {64,128,256,512,1024}");
  const auto dev = x.device();
  auto on_dev = [&](const Tensor& t, at::ScalarType dt, const char* name, const char* what) {
    TORCH_CHECK(t.device() == dev && t.scalar_type() == dt && t.is_contiguous(), name, what);
  };
  on_dev(w, at::kBFloat16, "w", " must be a contiguous bf16 tensor on the device of x");
  TORCH_CHECK(w.numel() == k, "w must hold K elements");
  on_dev(bias, at::kBFloat16, "bias", " must be a contiguous bf16 tensor on the device of x");
  TORCH_CHECK(bias.numel() >= 1, "bias must hold one element");
  on_dev(labels, at::kFloat, "labels", " must be a contiguous fp32 tensor on the device of x");
  TORCH_CHECK(labels.numel() == batch, "labels must hold one value per row");
  on_dev(n_valid, at::kLong, "n_valid", " must be an int64 tensor on the device of x");
  TORCH_CHECK(n_valid.numel() == 1, "n_valid must be one int64 word");
  on_dev(probs, at::kFloat, "probs", " must be a contiguous fp32 tensor on the device of x");
  TORCH_CHECK(probs.numel() == batch, "probs must hold one value per row");
  on_dev(hist, at::kLong, "hist", " must be a contiguous int64 tensor on the device of x");
  // T - 1 buckets with T >= 2; the bucket scale T - 1 must be exact in fp32
  TORCH_CHECK(hist.dim() == 2 && hist.size(0) == 2 && hist.size(1) >= 1 &&
                  hist.size(1) <= (int64_t{1} << 24),
              "hist must be [2, T - 1] with 2 <= T <= 2^24 + 1");
  on_dev(loss_sum, at::kDouble, "loss_sum", " must be an fp64 tensor on the device of x");
  TORCH_CHECK(loss_sum.numel() == 1, "loss_sum must hold one element");
  on_dev(count, at::kLong, "count", " must be an int64 tensor on the device of x");
  TORCH_CHECK(count.numel() == 1, "count must hold one element");
  c10::cuda::CUDAGuard guard(dev);
  bool ok = de::launch_head_eval(x.data_ptr(), static_cast<int>(k), w.data_ptr(), bias.data_ptr(),
                                 labels.data_ptr<float>(), batch, n_valid.data_ptr<int64_t>(),
                                 probs.data_ptr<float>(), hist.data_ptr<int64_t>(),
                                 static_cast<int>(hist.size(1)), loss_sum.data_ptr<double>(),
                                 count.data_ptr<int64_t>(), sm_count(), cur_stream());
  TORCH_CHECK(ok, "head_eval supports K in {64,128,256,512,1024}");
  check_launch();
}

void dense_sgd(Tensor p32, Tensor p16, Tensor g32, const Tensor& lr, double grad_scale) {
  TORCH_CHECK(p32.is_cuda() && p32.scalar_type() == at::kFloat && g32.scalar_type() == at::kFloat &&
              p16.scalar_type() == at::kBFloat16 && lr.scalar_type() == at::kFloat);
  TORCH_CHECK(p32.numel() % 4 == 0 && p32.numel() == g32.numel() && p32.numel() == p16.numel());
  c10::cuda::CUDAGuard guard(p32.device());
  de::launch_sgd_update(p32.data_ptr<float>(), p16.data_ptr(), g32.data_ptr<float>(),
                        lr.data_ptr<float>(), static_cast<float>(grad_scale), p32.numel(),
                        sm_count(), cur_stream());
  check_launch();
}

// Host checks shared by dense_adagrad / dense_adam: flat fp32 buffers (bf16 for p16) of one size,
// a multiple of 4 elements, 16-byte aligned (the kernel moves float4 / 4 x bf16); scalar device
// words for the learning rate and the step.  Messages carry strings only.
void check_dense_opt(const Tensor& p32, const Tensor& p16, const Tensor& g32,
                     const std::vector<std::pair<const Tensor*, const char*>>& state,
                     const Tensor& lr, const Tensor* step) {
  TORCH_CHECK(p32.is_cuda(), "p32 must be a CUDA tensor");
  const auto dev = p32.device();
  const int64_t n = p32.numel();
  TORCH_CHECK(n % 4 == 0, "the flat buffers must hold a multiple of 4 elements");
  auto flat = [&](const Tensor& t, at::ScalarType dt, const char* name, const char* what) {
    TORCH_CHECK(t.device() == dev && t.scalar_type() == dt, name, what);
    TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
    TORCH_CHECK(t.numel() == n, name, " must have as many elements as p32");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0, name,
                " must be 16-byte aligned");
  };
  flat(p32, at::kFloat, "p32", " must be an fp32 tensor");
  flat(p16, at::kBFloat16, "p16", " must be a bf16 tensor on the device of p32");
  flat(g32, at::kFloat, "g32", " must be an fp32 tensor on the device of p32");
  for (const auto& s : state)
    flat(*s.first, at::kFloat, s.second, " must be an fp32 tensor on the device of p32");
  auto word = [&](const Tensor& t, const char* name) {
    TORCH_CHECK(t.device() == dev && t.scalar_type() == at::kFloat && t.numel() == 1, name,
                " must be a one-element fp32 tensor on the device of p32");
  };
  word(lr, "lr");
  if (step != nullptr) word(*step, "step");
}

void dense_adagrad(Tensor p32, Tensor p16, Tensor g32, Tensor acc, const Tensor& lr, double eps) {
  check_dense_opt(p32, p16, g32, {{&acc, "acc"}}, lr, nullptr);
  c10::cuda::CUDAGuard guard(p32.device());
  de::launch_dense_opt(de::kOptAdagrad, p32.data_ptr<float>(), p16.data_ptr(),
                       g32.data_ptr<float>(), acc.data_ptr<float>(), nullptr,
                       lr.data_ptr<float>(), nullptr, 0.f, 0.f, static_cast<float>(eps),
                       p32.numel(), sm_count(), cur_stream());
  check_launch();
}

void dense_adam(Tensor p32, Tensor p16, Tensor g32, Tensor m, Tensor v, const Tensor& lr,
                const Tensor& step, double beta1, double beta2, double eps) {
  check_dense_opt(p32, p16, g32, {{&m, "m"}, {&v, "v"}}, lr, &step);
  c10::cuda::CUDAGuard guard(p32.device());
  de::launch_dense_opt(de::kOptAdam, p32.data_ptr<float>(), p16.data_ptr(),
                       g32.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                       lr.data_ptr<float>(), step.data_ptr<float>(), static_cast<float>(beta1),
                       static_cast<float>(beta2), static_cast<float>(eps), p32.numel(),
                       sm_count(), cur_stream());
  check_launch();
}

void cast_pad(const Tensor& src, Tensor dst) {
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kFloat && src.is_contiguous());
  TORCH_CHECK(dst.scalar_type() == at::kBFloat16 && dst.is_contiguous() &&
              dst.size(0) == src.size(0) && dst.size(1) >= src.size(1));
  c10::cuda::CUDAGuard guard(src.device());
  de::launch_cast_pad(src.data_ptr<float>(), static_cast<int>(src.size(1)), dst.data_ptr(),
                      static_cast<int>(dst.size(1)), src.size(0), cur_stream());
  check_launch();
}

// out[M,N] = act(a[M,K] @ b[N,K]^T + bias) on the hand-written wgmma kernel
void gemm_tn_bias_act(const Tensor& a, const Tensor& b, const c10::optional<Tensor>& bias,
                      Tensor out, bool relu, int64_t block_n) {
  check_bf16_2d(a, "a");
  check_bf16_2d(b, "b");
  check_bf16_2d(out, "out");
  TORCH_CHECK(a.size(1) == b.size(1) && out.size(0) == a.size(0) && out.size(1) == b.size(0),
              "shape mismatch");
  if (bias.has_value())
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() &&
                bias->numel() == b.size(0));
  c10::cuda::CUDAGuard guard(a.device());
  bool ok = de::launch_gemm_tn_bias_act(
      a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
      bias.has_value() ? bias->data_ptr() : nullptr, out.data_ptr(), out.stride(0),
      static_cast<int>(a.size(0)), static_cast<int>(b.size(0)), static_cast<int>(a.size(1)), relu,
      static_cast<int>(block_n), sm_count(), cur_stream());
  TORCH_CHECK(ok, "gemm_tn_bias_act: unsupported shape/alignment or launch failure");
  check_launch();
}

// dx[M,N] = (dy[M,K] @ wt[N,K]^T) * (act > 0); colsum[n] += column sums of dx  (one kernel)
void gemm_dgrad_relu_bias(const Tensor& dy, const Tensor& wt, const Tensor& act, Tensor dx,
                          Tensor colsum, int64_t block_n) {
  check_bf16_2d(dy, "dy");
  check_bf16_2d(wt, "wt");
  check_bf16_2d(act, "act");
  check_bf16_2d(dx, "dx");
  TORCH_CHECK(dy.size(1) == wt.size(1) && dx.size(0) == dy.size(0) && dx.size(1) == wt.size(0) &&
              act.size(0) == dx.size(0) && act.size(1) == dx.size(1), "shape mismatch");
  TORCH_CHECK(colsum.is_cuda() && colsum.scalar_type() == at::kFloat &&
              colsum.numel() >= dx.size(1));
  c10::cuda::CUDAGuard guard(dy.device());
  bool ok = de::launch_gemm_tn_fused(
      dy.data_ptr(), dy.stride(0), wt.data_ptr(), wt.stride(0), nullptr, dx.data_ptr(),
      dx.stride(0), static_cast<int>(dy.size(0)), static_cast<int>(wt.size(0)),
      static_cast<int>(dy.size(1)), 2, act.data_ptr(), act.stride(0), colsum.data_ptr<float>(),
      static_cast<int>(block_n), sm_count(), cur_stream());
  TORCH_CHECK(ok, "gemm_dgrad_relu_bias: unsupported shape/alignment or launch failure");
  check_launch();
}

// ------------------------------------------------------------------ symmetric memory (IPC)
// Buffers that peers map must not come from the caching allocator (its blocks are sub-ranges
// of larger cudaMalloc segments), so they are cudaMalloc'd here and wrapped with from_blob.
Tensor symm_alloc(int64_t nbytes, int64_t device_index) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device_index));
  void* ptr = nullptr;
  const size_t padded = (static_cast<size_t>(nbytes) + 255) & ~static_cast<size_t>(255);
  DE_CUDA_CHECK(cudaMalloc(&ptr, padded));
  DE_CUDA_CHECK(cudaMemset(ptr, 0, padded));
  DE_CUDA_CHECK(cudaDeviceSynchronize());
  auto deleter = [](void* p) { cudaFree(p); };
  return at::from_blob(ptr, {static_cast<int64_t>(padded)}, deleter,
                       at::TensorOptions()
                           .device(at::Device(at::kCUDA, static_cast<c10::DeviceIndex>(device_index)))
                           .dtype(at::kByte));
}

Tensor ipc_get_handle(const Tensor& buf) {
  TORCH_CHECK(buf.is_cuda());
  cudaIpcMemHandle_t h;
  DE_CUDA_CHECK(cudaIpcGetMemHandle(&h, buf.data_ptr()));
  Tensor out = at::empty({static_cast<int64_t>(sizeof(h))}, at::TensorOptions().dtype(at::kByte));
  std::memcpy(out.data_ptr(), &h, sizeof(h));
  return out;
}

int64_t ipc_open(const Tensor& handle, int64_t device_index) {
  TORCH_CHECK(!handle.is_cuda() && handle.numel() == sizeof(cudaIpcMemHandle_t));
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device_index));
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle.data_ptr(), sizeof(h));
  void* ptr = nullptr;
  DE_CUDA_CHECK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return reinterpret_cast<int64_t>(ptr);
}

void ipc_close(int64_t ptr, int64_t device_index) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device_index));
  cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr));
}

// ------------------------------------------------------------------ offload cache
// cache = [weight, state0, state1, tags, ticks, dirty, tick_word, stats] (absent states: empty
// tensors); host = device-visible pointers of [weight, state0, state1] of the host table.
de::CacheTable to_cache(at::TensorList cache, at::IntArrayRef host, int64_t n_sets,
                        int64_t n_spill, int64_t rows) {
  TORCH_CHECK(cache.size() == 8, "offload cache: 8 tensors expected");
  TORCH_CHECK(host.size() == 3, "offload cache: 3 host pointers expected");
  TORCH_CHECK(n_sets >= 1 && n_sets < (int64_t(1) << 31) && n_spill >= 0 && rows >= 1 &&
                  rows < (int64_t(1) << 32) - 1,
              "offload cache: bad geometry (n_sets ", n_sets, ", n_spill ", n_spill, ", rows ",
              rows, ")");
  const int64_t slots = n_sets * 32 + n_spill;
  const Tensor& w = cache[0];
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.is_contiguous() && w.dim() == 2 &&
                  w.size(0) == slots && w.size(1) >= 1 && w.data_ptr() != nullptr,
              "offload cache: weight must be a contiguous fp32 CUDA tensor [", slots, ", width]");
  TORCH_CHECK(w.size(1) % 4 != 0 || (reinterpret_cast<uintptr_t>(w.data_ptr()) % 16 == 0 &&
                                     host[0] % 16 == 0),
              "offload cache: rows of width % 4 == 0 must be 16-byte aligned");
  TORCH_CHECK(host[0] != 0, "offload cache: host table pointer is null");
  de::CacheTable T{};
  T.weight = w.data_ptr<float>();
  T.host_weight = reinterpret_cast<float*>(host[0]);
  T.width = static_cast<int32_t>(w.size(1));
  float** cs[2] = {&T.state0, &T.state1};
  float** hs[2] = {&T.host_state0, &T.host_state1};
  int32_t* sw[2] = {&T.state0_width, &T.state1_width};
  for (int k = 0; k < 2; ++k) {
    const Tensor& s = cache[1 + k];
    if (s.numel() == 0) {
      TORCH_CHECK(host[1 + k] == 0, "offload cache: host state without a cache state");
      continue;
    }
    TORCH_CHECK(s.is_cuda() && s.scalar_type() == at::kFloat && s.is_contiguous() &&
                    s.size(0) == slots && (s.dim() == 1 || (s.dim() == 2 && s.size(1) == w.size(1))),
                "offload cache: state must be fp32 CUDA [slots] or [slots, width]");
    TORCH_CHECK(host[1 + k] != 0 && host[1 + k] % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(s.data_ptr()) % 16 == 0,
                "offload cache: host state pointer is null or misaligned");
    *cs[k] = s.data_ptr<float>();
    *hs[k] = reinterpret_cast<float*>(host[1 + k]);
    *sw[k] = static_cast<int32_t>(s.dim() == 1 ? 1 : s.size(1));
  }
  auto check_i = [&](const Tensor& t, at::ScalarType ty, int64_t n, const char* what) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == ty && t.is_contiguous() && t.numel() == n &&
                    t.device() == w.device(),
                "offload cache: ", what, " must be a contiguous CUDA tensor of ", n, " elements");
  };
  check_i(cache[3], at::kLong, slots, "tags (int64)");
  check_i(cache[4], at::kInt, n_sets * 32, "ticks (int32)");
  check_i(cache[5], at::kInt, slots, "dirty (int32)");
  check_i(cache[6], at::kInt, 1, "tick_word (int32)");
  check_i(cache[7], at::kLong, 4, "stats (int64)");
  T.tags = cache[3].data_ptr<int64_t>();
  T.ticks = cache[4].data_ptr<int32_t>();
  T.dirty = cache[5].data_ptr<int32_t>();
  T.tick_word = cache[6].data_ptr<int32_t>();
  T.stats = cache[7].data_ptr<int64_t>();
  T.n_sets = n_sets;
  T.n_spill = n_spill;
  T.rows = rows;
  return T;
}

// One cache pass of one table (see offload_cache.cu).  descs / tables: the table's cached inputs
// on their *host* rows (local_table 0, item_off rebased to [0, n_items)) and one TableDesc with
// key_base 0; remap: their CacheRemap records (device bytes); out_ptr: the slot-id buffer.
void offload_cache_pass(at::TensorList cache, at::IntArrayRef host, int64_t n_sets,
                        int64_t n_spill, int64_t rows, const Tensor& descs, const Tensor& tables,
                        int64_t n_inputs, int64_t batch, bool ids64, int64_t n_items,
                        bool prefill_sentinel, const Tensor& remap, int64_t n_remap,
                        int64_t max_remap_n, int64_t out_ptr, bool train) {
  de::CacheTable T = to_cache(cache, host, n_sets, n_spill, rows);
  TORCH_CHECK(n_items == n_spill && n_items >= 1,
              "offload cache: the spill region must hold every id of the step (", n_items,
              " ids, ", n_spill, " spill slots)");
  TORCH_CHECK(n_items < (int64_t(1) << 31), "offload cache: too many ids per step");
  TORCH_CHECK(descs.is_cuda() && tables.is_cuda() && remap.is_cuda() &&
                  descs.device() == cache[0].device() && remap.device() == cache[0].device(),
              "offload cache: descriptors must live on the cache's GPU");
  TORCH_CHECK(descs.numel() == n_inputs * static_cast<int64_t>(sizeof(de::InputDesc)) &&
                  tables.numel() == static_cast<int64_t>(sizeof(de::TableDesc)) &&
                  remap.numel() == n_remap * static_cast<int64_t>(sizeof(de::CacheRemap)) &&
                  n_inputs >= 1 && n_remap >= 1 && max_remap_n >= 0,
              "offload cache: descriptor array sizes do not match their counts");
  TORCH_CHECK(out_ptr != 0 && out_ptr % (ids64 ? 8 : 4) == 0, "offload cache: bad slot-id buffer");
  TORCH_CHECK(n_sets * 32 + n_spill < (ids64 ? (int64_t(1) << 62) : (int64_t(1) << 31)),
              "offload cache: slot ids do not fit the id type");
  c10::cuda::CUDAGuard guard(cache[0].device());
  auto stream = cur_stream();
  auto dev = cache[0].device();
  auto i64 = at::TensorOptions().device(dev).dtype(at::kLong);
  auto i32 = at::TensorOptions().device(dev).dtype(at::kInt);
  // nothing above launches: every argument is checked before the first kernel
  de::launch_cache_spill_writeback(T, sm_count(), stream);
  check_launch();
  auto sorted = sort_items(descs, tables, 1, n_inputs, batch, batch, {}, ids64, n_items, rows,
                           prefill_sentinel);
  const Tensor& keys = std::get<0>(sorted);
  const Tensor& seg_start = std::get<2>(sorted);
  const Tensor& n_unique = std::get<3>(sorted);
  Tensor uniq = at::empty({n_items}, i64), slot_of = at::empty({n_items}, i64);
  Tensor move = at::empty({n_items}, i64);
  Tensor set_a = at::empty({n_items}, i32), item_a = at::empty({n_items}, i32);
  Tensor set_b = at::empty({n_items}, i32), item_b = at::empty({n_items}, i32);
  Tensor set_sorted = at::empty({n_items}, i64);
  Tensor seg = at::empty({n_items + 1}, i64), n_seg = at::zeros({1}, i64);
  const size_t temp_bytes =
      std::max(de::radix_sort_temp_bytes(n_items), de::head_segments_temp_bytes(n_items));
  Tensor temp = at::empty({static_cast<int64_t>(temp_bytes)},
                          at::TensorOptions().device(dev).dtype(at::kByte));
  de::launch_cache_probe(T, keys.data_ptr<int64_t>(), seg_start.data_ptr<int64_t>(),
                         n_unique.data_ptr<int64_t>(), n_items, train, uniq.data_ptr<int64_t>(),
                         reinterpret_cast<uint32_t*>(set_a.data_ptr<int>()),
                         reinterpret_cast<uint32_t*>(item_a.data_ptr<int>()),
                         slot_of.data_ptr<int64_t>(), move.data_ptr<int64_t>(), sm_count(), stream);
  check_launch();
  // stable sort by set: a set's misses keep their ascending row order
  int where = de::radix_sort_pairs32(
      temp.data_ptr(), reinterpret_cast<uint32_t*>(set_a.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(item_a.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(set_b.data_ptr<int>()),
      reinterpret_cast<uint32_t*>(item_b.data_ptr<int>()), set_sorted.data_ptr<int64_t>(), n_items,
      bit_length(n_sets), stream);
  const Tensor& u_sorted = where == 0 ? item_a : item_b;
  de::head_segments(temp.data_ptr(), set_sorted.data_ptr<int64_t>(), n_items,
                    seg.data_ptr<int64_t>(), n_seg.data_ptr<int64_t>(), stream);
  check_launch();
  de::launch_cache_assign(T, set_sorted.data_ptr<int64_t>(),
                          reinterpret_cast<const uint32_t*>(u_sorted.data_ptr<int>()),
                          seg.data_ptr<int64_t>(), n_seg.data_ptr<int64_t>(), n_items, train,
                          uniq.data_ptr<int64_t>(), slot_of.data_ptr<int64_t>(),
                          move.data_ptr<int64_t>(), sm_count(), stream);
  check_launch();
  de::launch_cache_fill(T, n_unique.data_ptr<int64_t>(), n_items, uniq.data_ptr<int64_t>(),
                        slot_of.data_ptr<int64_t>(), move.data_ptr<int64_t>(), sm_count(), stream);
  check_launch();
  de::launch_cache_remap(reinterpret_cast<const de::CacheRemap*>(remap.data_ptr()),
                         static_cast<int>(n_remap), max_remap_n, uniq.data_ptr<int64_t>(),
                         n_unique.data_ptr<int64_t>(), slot_of.data_ptr<int64_t>(), rows, ids64,
                         reinterpret_cast<void*>(out_ptr), sm_count(), stream);
  check_launch();
}

void offload_cache_flush(at::TensorList cache, at::IntArrayRef host, int64_t n_sets,
                         int64_t n_spill, int64_t rows) {
  de::CacheTable T = to_cache(cache, host, n_sets, n_spill, rows);
  c10::cuda::CUDAGuard guard(cache[0].device());
  de::launch_cache_flush(T, sm_count(), cur_stream());
  check_launch();
}

// Map a host tensor's storage for zero-copy GPU access (CPU-offloaded tables): returns the
// device-visible pointer of pinned (cudaHostRegister'ed / pin_memory) memory.
int64_t host_device_pointer(const Tensor& host) {
  TORCH_CHECK(!host.is_cuda());
  void* dptr = nullptr;
  DE_CUDA_CHECK(cudaHostGetDevicePointer(&dptr, host.data_ptr(), 0));
  return reinterpret_cast<int64_t>(dptr);
}

}  // namespace

TORCH_LIBRARY(de_b200, m) {
  m.def("struct_sizes() -> int[]", &struct_sizes);
  m.def(
      "sync_ctx_create(int[] flag_ptrs, Tensor state, int rank, int world, int timeout_cycles, "
      "int error_ptr) -> int",
      &sync_ctx_create);
  m.def("sync_only(int[] sync) -> ()", &sync_only);
  m.def(
      "lookup_fwd(Tensor descs, int n_inputs, int batch, int src_batch, int dst_batch, "
      "int dst_stride, int[] src_ptrs, int[] dst_ptrs, int rot, bool ids64, int act_dtype, "
      "bool vec4, int[] sync, int tile_samples, int table_dtype=0, bool vec8=False) -> ()",
      &lookup_fwd);
  m.def(
      "scatter_add_bwd(Tensor descs, int n_inputs, int batch, int src_batch, int grad_batch, "
      "int grad_stride, int[] src_ptrs, int[] grad_ptrs, int rot, float scale, int scale_ptr, bool ids64, "
      "int act_dtype, bool vec4, bool vec8, int[] sync, bool staged) -> ()",
      &scatter_add_bwd);
  m.def(
      "sort_items(Tensor descs, Tensor tables, int n_tables, int n_inputs, int batch, "
      "int src_batch, int[] src_ptrs, bool ids64, int n_items, int total_rows, "
      "bool prefill_sentinel) -> "
      "(Tensor, Tensor, Tensor, Tensor)",
      &sort_items);
  m.def("radix_sort_pairs(Tensor keys, Tensor items, int end_bit) -> (Tensor, Tensor)",
        &radix_sort_pairs);
  m.def("radix_sort_pairs32(Tensor keys, Tensor items, int end_bit) -> (Tensor, Tensor)",
        &radix_sort_pairs32);
  m.def("head_segments(Tensor sorted_keys) -> (Tensor, Tensor)", &head_segments);
  m.def(
      "segment_update(Tensor descs, Tensor tables, int n_tables, int batch, int grad_batch, "
      "int grad_stride, int[] grad_ptrs, Tensor sorted_keys, Tensor sorted_items, "
      "Tensor seg_start, Tensor n_unique, int opt_kind, float lr, float eps, float beta1, "
      "float beta2, float bias1, float bias2, float grad_scale, float weight_decay, int lr_ptr, "
      "Tensor? emit_keys, Tensor? emit_rows, int max_width, int act_dtype, bool vec4, "
      "Tensor? scratch, int step_ptr, int table_dtype=0, int state_dtype=0, "
      "float lr_power=-0.5, float l1=0., float l2=0., float l2_shrinkage=0., "
      "float ftrl_beta=0.) -> ()",
      &segment_update);
  m.def(
      "embedding_lookup_fwd(Tensor param, Tensor values, Tensor? offsets, int hotness, int batch, "
      "int combiner, bool out_bf16) -> Tensor",
      &embedding_lookup_fwd);
  m.def(
      "embedding_scatter_add(Tensor(a!) dst, Tensor values, Tensor? offsets, int hotness, "
      "int batch, int combiner, Tensor grad, float scale) -> ()",
      &embedding_scatter_add);
  m.def(
      "embedding_lookup_grad(Tensor values, Tensor? offsets, int hotness, int batch, int combiner, "
      "Tensor grad, int num_rows) -> (Tensor, Tensor)",
      &embedding_lookup_grad);
  m.def("row_to_split(Tensor indices, int num_rows) -> Tensor", &row_to_split);
  m.def("hash_init(Tensor(a!) table) -> ()", &hash_init);
  m.def(
      "integer_lookup(Tensor(a!) table, Tensor(b!) count, Tensor(c!) next_index, Tensor keys, "
      "int capacity) -> Tensor",
      &integer_lookup);
  m.def(
      "barrier(int[] flag_ptrs, Tensor(a!) epoch, int rank, int world, int channel, "
      "int timeout_cycles, int error_ptr) -> ()",
      &barrier);
  m.def(
      "allreduce(int[] buf_ptrs, int[] flag_ptrs, Tensor(a!) epoch, int rank, int world, "
      "int n_elems, float scale, bool bf16, int channel, int timeout_cycles, "
      "int error_ptr, int mc_ptr, int max_blocks) -> ()",
      &allreduce);
  m.def("gather_segments(Tensor segs, int[] src_ptrs, Tensor(a!) dst, int max_seg_elems) -> ()",
        &gather_segments);
  m.def(
      "p2p_store_bench(Tensor src, int dst_ptr, int n_rows, int row_bytes, int vec_bytes, "
      "int dst_stride, int unroll, int blocks, int threads) -> ()",
      &p2p_store_bench);
  m.def(
      "push_segments(Tensor segs, Tensor src, int[] dst_ptrs, int max_seg_elems, int[] sync) -> ()",
      &push_segments);
  m.def(
      "push_grad(Tensor routes, int n_routes, Tensor src, int dst_dtype, float scale, int[] sync) "
      "-> ()",
      &push_grad);
  m.def(
      "stream_push(int[] src_ptrs, int[] dst_ptrs, int[] row_bytes, Tensor counters, "
      "int chunk_rows, int rows, int blocks, int[] sync) -> ()",
      &stream_push);
  m.def(
      "rowslice_reduce(Tensor partial, int out_ptr, int out_stride, int out_dtype, Tensor cols) "
      "-> ()",
      &rowslice_reduce);
  m.def(
      "gather_ragged(Tensor segs, int[] val_ptrs, int[] split_ptrs, Tensor(a!) dst_vals, "
      "Tensor(b!) goff, int b, int max_cap) -> ()",
      &gather_ragged);
  m.def("select_copy(Tensor[] src0, Tensor[] src1, Tensor(a!)[] dst, Tensor slot_flag) -> ()",
        &select_copy);
  m.def("copy_cast_2d(Tensor src, int dst_ptr, int dst_stride, int dst_dtype, float scale) -> ()",
        &copy_cast_2d);
  m.def("interact_fwd(Tensor bottom, Tensor emb, int n_emb, Tensor(a!) z, int[] sync) -> ()",
        &interact_fwd);
  m.def(
      "interact_bwd(Tensor bottom, Tensor emb, int n_emb, Tensor dz, Tensor(a!) dbottom, "
      "int demb_ptr, int demb_stride, float emb_grad_scale, Tensor? routes, int n_routes, "
      "int[] sync, Tensor? done_counters, int chunk_rows, Tensor? apply_descs=None, "
      "float apply_scale=0.0, int apply_scale_ptr=0, bool apply_ids64=False) -> ()",
      &interact_bwd);
  m.def("avgpool_fwd(Tensor x, int n, Tensor(a!) out, int stride) -> ()", &avgpool_fwd);
  m.def("avgpool_bwd(Tensor dout, Tensor(a!) dx, int n, int stride) -> ()", &avgpool_bwd);
  m.def("relu_bwd_bias(Tensor(a!) dy, Tensor y, Tensor(b!) db) -> ()", &relu_bwd_bias);
  m.def("cross_fwd(Tensor x0, Tensor s, Tensor xl, Tensor(a!) out) -> ()", &cross_fwd);
  m.def("cross_bwd(Tensor dy, Tensor x0, Tensor(a!) g, Tensor(b!) db) -> ()", &cross_bwd);
  m.def(
      "cross_dx0(Tensor d_chain, Tensor[] dy, Tensor[] s, Tensor(a!) dx0, Tensor(b!) d_bottom) "
      "-> ()",
      &cross_dx0);
  m.def(
      "head_loss(Tensor x, Tensor w, Tensor bias, Tensor labels, float inv_batch, Tensor(a!) dx, "
      "Tensor(b!) dw, Tensor(c!) db, Tensor(d!) dbias_prev, Tensor(e!) loss_sum, Tensor? logits) "
      "-> ()",
      &head_loss);
  m.def(
      "head_eval(Tensor x, Tensor w, Tensor bias, Tensor labels, Tensor n_valid, Tensor(a!) probs, "
      "Tensor(b!) hist, Tensor(c!) loss_sum, Tensor(d!) count) -> ()",
      &head_eval);
  m.def(
      "dense_sgd(Tensor(a!) p32, Tensor(b!) p16, Tensor(c!) g32, Tensor lr, float grad_scale) "
      "-> ()",
      &dense_sgd);
  m.def(
      "dense_adagrad(Tensor(a!) p32, Tensor(b!) p16, Tensor(c!) g32, Tensor(d!) acc, Tensor lr, "
      "float eps) -> ()",
      &dense_adagrad);
  m.def(
      "dense_adam(Tensor(a!) p32, Tensor(b!) p16, Tensor(c!) g32, Tensor(d!) m, Tensor(e!) v, "
      "Tensor lr, Tensor step, float beta1, float beta2, float eps) -> ()",
      &dense_adam);
  m.def("cast_pad(Tensor src, Tensor(a!) dst) -> ()", &cast_pad);
  m.def(
      "gemm_tn_bias_act(Tensor a, Tensor b, Tensor? bias, Tensor(a!) out, bool relu, int block_n) "
      "-> ()",
      &gemm_tn_bias_act);
  m.def(
      "gemm_dgrad_relu_bias(Tensor dy, Tensor wt, Tensor act, Tensor(a!) dx, Tensor(b!) colsum, "
      "int block_n) -> ()",
      &gemm_dgrad_relu_bias);
  m.def("symm_alloc(int nbytes, int device_index) -> Tensor", &symm_alloc);
  m.def("ipc_get_handle(Tensor buf) -> Tensor", &ipc_get_handle);
  m.def("ipc_open(Tensor handle, int device_index) -> int", &ipc_open);
  m.def("ipc_close(int ptr, int device_index) -> ()", &ipc_close);
  m.def("host_device_pointer(Tensor host) -> int", &host_device_pointer);
  m.def(
      "offload_cache_pass(Tensor[] cache, int[] host, int n_sets, int n_spill, int rows, "
      "Tensor descs, Tensor tables, int n_inputs, int batch, bool ids64, int n_items, "
      "bool prefill_sentinel, Tensor remap, int n_remap, int max_remap_n, int out_ptr, "
      "bool train) -> ()",
      &offload_cache_pass);
  m.def("offload_cache_flush(Tensor[] cache, int[] host, int n_sets, int n_spill, int rows) -> ()",
        &offload_cache_flush);
}
