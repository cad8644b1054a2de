// Host-callable launchers of the sm_90a kernels. Plain C++ (no torch headers) so that the .cu
// files compile in seconds; bindings.cpp adapts these to TORCH_LIBRARY ops.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace de {

constexpr int kMaxPeers = 16;
// grid-stride elementwise kernels launch at most a few blocks per SM of an H100 SXM (132 SMs)
constexpr int kGridCapSms = 132;

// One entry per local input (feature) served by this rank. Resolved once from the sharding plan
// so a single persistent kernel handles every table of the rank (hundreds in the large models).
struct alignas(16) InputDesc {
  const void* table;       // base of the (fused) local table, row major [rows, width]; fp32,
                           // bf16 or fp16 (one storage type per launch: `table_dtype`)
  const void* ids;         // direct ids pointer, or nullptr -> src_ptrs[s] + ids_off
  const int64_t* offsets;  // CSR row_splits for ragged inputs, nullptr for fixed hotness
  int64_t ids_off;         // element offset of this input inside a source staging buffer
  int64_t id_shift;        // added to the raw id (row slices: -first_row)
  int64_t sub_rows;        // ids valid after the shift: [0, sub_rows); others contribute zero
  int64_t row_base;        // first row of this sub-table inside the fused table
  int32_t width;           // embedding width (columns)
  int32_t hotness;         // ids per sample for fixed hotness, 0 = ragged (use offsets)
  int32_t dst_col;         // first column in the destination (requester output / grad) row
  int32_t combiner;        // 0 = sum, 1 = mean
  int32_t local_table;     // index into the rank's TableDesc array
  int32_t flags;           // bit 0: skip the store when the sample has no id inside this shard
  int64_t item_off;        // first (key, item) slot of this input in the sorted-update arrays
};

struct PeerPtrs {
  void* p[kMaxPeers];
};

// Cross-GPU producer/consumer signalling folded into the data kernels (no separate barrier
// launches): a kernel may *wait* at its head for the peers' signals on one channel and *signal*
// all peers from its tail once every block has finished.  Flags are per (channel, writer)
// epoch words in the peer-mapped signal pad; the epochs a rank expects / publishes live in
// device memory (`state`), so a captured CUDA graph replays without host patching.
//   state[0..15]   wait epochs   (signals consumed per channel)
//   state[16..31]  signal epochs (signals published per channel)
//   state[32..63]  block counters (one per call site: `counter_slot`)
constexpr int kSyncChannels = 16;
constexpr int kSyncStateWords = 64;
struct SyncArgs {
  PeerPtrs flags;               // signal pads of all ranks (peer mapped)
  uint32_t* state;              // this rank's epoch / counter words (nullptr = no signalling)
  int* error_flag;              // host-mapped watchdog word (may be nullptr)
  unsigned long long timeout;   // cycles before a wait gives up and traps (0 = wait forever)
  int32_t rank, world;
  int32_t wait_ch;              // >= 0: wait until every peer's flag >= wait epoch + 1
  int32_t wait_abs_ch;          // >= 0: wait until every peer's flag >= this rank's *signal*
                                //       epoch of that channel (peers have caught up with me)
  int32_t signal_ch;            // >= 0: publish signal epoch + 1 to every peer at the tail
  int32_t counter_slot;         // block counter used by this launch (unique per call site)
};
inline SyncArgs no_sync() {
  SyncArgs s{};
  s.state = nullptr;
  s.wait_ch = s.wait_abs_ch = s.signal_ch = -1;
  return s;
}

// One contiguous piece of a requester-side gradient row and where it goes on its owner:
// columns [src_col, src_col + width) of local sample i land at
// dst + i * dst_stride + dst_col (dst already points at this requester's row block of the
// owner's receive buffer; peer mapped).
struct alignas(16) GradRoute {
  void* dst;
  int64_t dst_stride;  // elements
  int32_t src_col;
  int32_t width;
  int32_t dst_col;
  int32_t pad;
};

enum OptimizerKind : int32_t {
  kOptSGD = 0,
  kOptAdagrad = 1,
  kOptRowwiseAdagrad = 2,
  kOptAdam = 3,
  kOptEmit = 4,
  kOptRowwiseAdam = 5,  // Adam with element-wise m (state0) and one fp32 v word per row (state1)
  kOptFtrl = 6,         // FTRL-Proximal: accumulator n (state0) and linear term z (state1)
  kOptMomentum = 7,     // momentum SGD: element-wise momentum buffer b (state0)
};

// One entry per (fused) local table, used by the sorted/deduplicated update path.
struct alignas(16) TableDesc {
  void* weight;       // [rows, width]; fp32, bf16 or fp16 (`table_dtype` of the launch)
  void* state0;       // Adagrad accumulator [rows,width] / row-wise [rows] / Adam m / row-wise
                      // Adam m / FTRL n / momentum b
  void* state1;       // Adam v / row-wise Adam v [rows] / FTRL z  (element-wise state: fp32 or bf16,
                      // `state_dtype` of the launch; row-wise state is always fp32)
  int64_t rows;
  int64_t key_base;   // first global row key of this table (prefix sum of rows)
  int32_t width;
  int32_t pad;
};

struct OptimizerArgs {
  int32_t kind;
  float lr;
  float eps;
  float beta1, beta2;
  float bias1, bias2;  // Adam bias corrections 1-beta^t
  float grad_scale;    // applied to the summed gradient (1/world for the global-mean contract)
  float weight_decay;
  const float* lr_ptr;  // optional device-resident learning rate (overrides lr; graph replay safe)
  const float* step_ptr;  // optional device-resident Adam step count t (bias1/bias2 are then
                          // recomputed as 1 - beta^t on the device; graph replay safe); it
                          // also keys the stochastic rounding of 16-bit tables
  // FTRL-Proximal (kind kOptFtrl; the other kinds ignore them): P(n) = n^(-lr_power)
  float lr_power;
  float l1, l2;
  float l2_shrinkage;
  float ftrl_beta;     // Keras's beta: adds beta / (2 lr) to l2
  // kWeightDecayL2: weight_decay * w joins the gradient; kWeightDecayDecoupled (AdamW): the
  // weight is scaled by 1 - lr * weight_decay and the step comes from the undecayed gradient
  int32_t weight_decay_mode;
  // momentum SGD (kind kOptMomentum; the other kinds ignore them), torch.optim.SGD's buffer:
  // b = momentum * b + g, then w -= lr * b, or with nesterov w -= lr * (momentum * b + g).
  // Appended so that the offsets of the fields above stay put.
  float momentum;
  int32_t nesterov;
};

constexpr int kWeightDecayL2 = 0;
constexpr int kWeightDecayDecoupled = 1;

// ---- pooled lookup forward (+ optional fused push to peer output buffers) ------------------
// ids come from src.p[g / src_batch] (peer mapped) or desc.ids; pooled rows are stored to
// dst.p[g / dst_batch] + (g % dst_batch) * dst_stride + dst_col.
// act_dtype: 0 = fp32, 1 = bf16, 2 = fp16 (dtype of the activations / gradients on the wire)
// table_dtype: storage of every table of the launch, same codes; rows are pooled in fp32.
// vec8 (16-bit tables with vec4 only): every width, destination column and row stride is a
// multiple of 8, so a lane loads 8 columns (16 bytes) at a time.
void launch_lookup_fwd(const InputDesc* descs, int n_inputs, int64_t batch, int64_t src_batch,
                       int64_t dst_batch, int64_t dst_stride, const PeerPtrs& src,
                       const PeerPtrs& dst, int rot, bool ids64, int act_dtype, bool vec4,
                       int sm_count, cudaStream_t stream, const SyncArgs& sync,
                       int tile_samples = 32, int table_dtype = 0, bool vec8 = false);

// ---- backward: atomic scatter-add of (scaled) gradient rows into the table (SGD fast path,
// also used to build dense gradients of replicated tables).  fp32 tables only. Gradient rows are pulled from
// grad.p[g / grad_batch] + (g % grad_batch) * grad_stride + dst_col (peer mapped).
void launch_scatter_add_bwd(const InputDesc* descs, int n_inputs, int64_t batch, int64_t src_batch,
                            int64_t grad_batch, int64_t grad_stride, const PeerPtrs& src,
                            const PeerPtrs& grad, int rot, float scale, const float* scale_ptr,
                            bool ids64, int act_dtype, bool vec4, int sm_count,
                            cudaStream_t stream, bool vec8, const SyncArgs& sync,
                            bool staged = false);

// ---- backward: sorted / deduplicated path -----------------------------------------------
// keys32: `keys` points at uint32 keys (every key incl. the sentinel fits 32 bits)
void launch_build_keys(const InputDesc* descs, const TableDesc* tables, int n_tables, int n_inputs,
                       int64_t batch, int64_t src_batch, const PeerPtrs& src, bool ids64, void* keys,
                       uint32_t* items, int sm_count, cudaStream_t stream, bool keys32 = false);
size_t sort_pairs_temp_bytes(int64_t n);
void sort_pairs(void* temp, size_t temp_bytes, const int64_t* keys_in, int64_t* keys_out,
                const uint32_t* items_in, uint32_t* items_out, int64_t n, int end_bit,
                cudaStream_t stream);
size_t unique_temp_bytes(int64_t n);
// seg_start[u] = first sorted position of unique key u; *n_unique on device; seg_start[n_unique] = n
void unique_segments(void* temp, size_t temp_bytes, const int64_t* sorted_keys, int64_t n,
                     int64_t* seg_start, int64_t* n_unique, cudaStream_t stream);
// first-party replacements of the two CUB calls above (radix_sort.cu); DE_B200_SORT=own selects them
size_t radix_sort_temp_bytes(int64_t n);
int radix_sort_pairs(void* temp, int64_t* keys_a, uint32_t* items_a, int64_t* keys_b,
                     uint32_t* items_b, int64_t n, int end_bit, cudaStream_t stream);
int radix_sort_pairs32(void* temp, uint32_t* keys_a, uint32_t* items_a, uint32_t* keys_b,
                       uint32_t* items_b, int64_t* keys_out64, int64_t n, int end_bit,
                       cudaStream_t stream);
// keys only, sorted in place between keys_a and keys_b; returns 0 (sorted in a) or 1 (in b)
int radix_sort_keys32(void* temp, uint32_t* keys_a, uint32_t* keys_b, int64_t n, int end_bit,
                      cudaStream_t stream);
size_t head_segments_temp_bytes(int64_t n);
void head_segments(void* temp, const int64_t* sorted_keys, int64_t n, int64_t* seg_start,
                   int64_t* n_unique, cudaStream_t stream);
void launch_segment_update(const InputDesc* descs, const TableDesc* tables, int n_tables,
                           int64_t batch, int64_t grad_batch, int64_t grad_stride,
                           const PeerPtrs& grad, const int64_t* sorted_keys,
                           const uint32_t* sorted_items, const int64_t* seg_start,
                           const int64_t* n_unique, int64_t n_items, const OptimizerArgs& opt,
                           int64_t* emit_keys, float* emit_rows, int max_width, int act_dtype,
                           bool vec4, int sm_count, cudaStream_t stream, int table_dtype = 0,
                           int state_dtype = 0);
// state_dtype: storage of the Adagrad accumulator / Adam moments, 0 = fp32, 1 = bf16 (widened
// to fp32 for the update, stored with stochastic rounding; other optimizers ignore it).

bool launch_balanced_update(const InputDesc* descs, const TableDesc* tables, int n_tables,
                            int64_t batch, int64_t grad_batch, int64_t grad_stride,
                            const PeerPtrs& grad, const int64_t* sorted_keys,
                            const uint32_t* sorted_items, int64_t n_items,
                            const int64_t* seg_start, const int64_t* n_unique,
                            const OptimizerArgs& opt, float* scratch, int scratch_width,
                            int max_width, int act_dtype, int sm_count, cudaStream_t stream,
                            int table_dtype = 0, int state_dtype = 0);

// ---- HBM row cache of host-offloaded fp32 tables (offload_cache.cu) ------------------------
// Slots [0, n_sets * 32) are the sets (32 ways each), [n_sets * 32, + n_spill) the spill region.
struct CacheTable {
  float* weight;        // [slots, width] HBM
  float* state0;        // [slots, state0_width] HBM or nullptr
  float* state1;        // [slots, state1_width] HBM or nullptr
  float* host_weight;   // [rows, width] pinned host table (device-visible UVA pointer)
  float* host_state0;   // its optimizer state, same layout as the cache's
  float* host_state1;
  int64_t* tags;        // [slots]: host row held by the slot, -1 = empty
  int32_t* ticks;       // [n_sets * 32]: tick of the last use
  int32_t* dirty;       // [slots]: the slot was updated since it was filled / flushed
  int32_t* tick_word;   // last tick of a finished cache pass (device resident)
  int64_t* stats;       // hits, misses, spills, write-backs (unique rows)
  int64_t n_sets;
  int64_t n_spill;
  int64_t rows;         // host rows (= the sentinel key of the pass's sort)
  int32_t width;
  int32_t state0_width;  // width, 1 (row-wise Adagrad) or 0
  int32_t state1_width;  // width (Adam v) or 0
  int32_t pad;
};
// One cached input of the remap: ids[0, n) + id_shift valid below sub_rows are host rows
// row_base + id; their slot ids go to out[out_off + i] (-1 for the others).
struct alignas(16) CacheRemap {
  const void* ids;
  int64_t n;
  int64_t id_shift;
  int64_t sub_rows;
  int64_t row_base;
  int64_t out_off;
};
void launch_cache_spill_writeback(const CacheTable& T, int sm_count, cudaStream_t stream);
void launch_cache_probe(const CacheTable& T, const int64_t* sorted_keys, const int64_t* seg_start,
                        const int64_t* n_unique, int64_t cap, bool train, int64_t* uniq,
                        uint32_t* miss_set, uint32_t* miss_item, int64_t* slot_of, int64_t* move,
                        int sm_count, cudaStream_t stream);
void launch_cache_assign(const CacheTable& T, const int64_t* set_sorted, const uint32_t* u_sorted,
                         const int64_t* seg, const int64_t* n_seg, int64_t cap, bool train,
                         const int64_t* uniq, int64_t* slot_of, int64_t* move, int sm_count,
                         cudaStream_t stream);
void launch_cache_fill(const CacheTable& T, const int64_t* n_unique, int64_t cap,
                       const int64_t* uniq, const int64_t* slot_of, const int64_t* move,
                       int sm_count, cudaStream_t stream);
void launch_cache_remap(const CacheRemap* inputs, int n_inputs, int64_t max_n,
                        const int64_t* uniq, const int64_t* n_unique, const int64_t* slot_of,
                        int64_t rows, bool ids64, void* out, int sm_count, cudaStream_t stream);
void launch_cache_flush(const CacheTable& T, int sm_count, cudaStream_t stream);

// ---- misc ---------------------------------------------------------------------------------
void launch_row_to_split(const int64_t* coo_indices, int64_t nnz, int64_t num_rows,
                         int64_t* row_splits, cudaStream_t stream);
void launch_hash_init(int64_t* table, int64_t n_slots, cudaStream_t stream);
void launch_integer_lookup(int64_t* table, int64_t n_slots, uint32_t* counts, int64_t* next_index,
                           const int64_t* keys, int64_t n, int64_t capacity, int64_t* out,
                           cudaStream_t stream);

// ---- communication kernels ----------------------------------------------------------------
// Flag barrier over peer-mapped signal pads: flags.p[r] points at rank r's pad (>= world slots
// of uint32 per channel); epoch lives in device memory so the kernel can be graph-replayed.
void launch_barrier(const PeerPtrs& flags, uint32_t* epoch, int rank, int world, int channel,
                    unsigned long long timeout_cycles, int* error_flag, cudaStream_t stream);
// Two-shot all-reduce (reduce-scatter + all-gather) over peer-mapped buffers, fused with scale.
void launch_allreduce(const PeerPtrs& bufs, const PeerPtrs& flags, uint32_t* epoch, int rank,
                      int world, int64_t n_elems, float scale, bool bf16, int channel,
                      unsigned long long timeout_cycles, int* error_flag, int sm_count,
                      cudaStream_t stream, int max_blocks = 0);
// Multimem (NVLS) variant: mc_ptr is the multicast mapping of the same symmetric buffer.
void launch_allreduce_multimem(void* mc_ptr, const PeerPtrs& flags, uint32_t* epoch, int rank,
                               int world, int64_t n_elems, float scale, bool bf16, int channel,
                               unsigned long long timeout_cycles, int* error_flag, int sm_count,
                               cudaStream_t stream, int max_blocks = 0);
// Micro-benchmark of kernel-issued row stores into (peer) memory, see comm_kernels.cu
void launch_p2p_store_bench(const void* src, void* dst, int64_t n_rows, int row_bytes,
                            int vec_bytes, int64_t dst_stride, int unroll, int blocks, int threads,
                            cudaStream_t stream);
// Standalone signalling kernel (one block): the wait / signal parts of `sync` without any data.
void launch_sync_only(const SyncArgs& sync, cudaStream_t stream);
// Segmented P2P *push* of index segments into the owners' id buffers (the reference's
// 'inp_dp_to_mp' all-to-all as fire-and-forget NVLink stores):
// segs[j] = {dst_rank, src_elem_off, dst_elem_off, n_elems}
void launch_push_segments(const int64_t* segs, int n_seg, const void* src, const PeerPtrs& dst,
                          int elem_bytes, int64_t max_seg_elems, int sm_count,
                          cudaStream_t stream, const SyncArgs& sync);
// Gradient all-to-all as a push: every route piece of the local gradient rows [rows, *] is cast
// to the wire dtype and stored into its owner's receive buffer.  src_dtype / dst_dtype: 0 fp32,
// 1 bf16, 2 fp16.
void launch_push_grad(const GradRoute* routes, int n_routes, const void* src, int64_t src_stride,
                      int src_dtype, int dst_dtype, int64_t rows, float scale, int sm_count,
                      cudaStream_t stream, const SyncArgs& sync);
// Streaming push of a locally staged, owner-major gradient buffer: block p of the staging
// buffer ([rows, row_bytes[p]] contiguous) goes to peer p's receive buffer.  The kernel follows
// the producer (e.g. the interaction backward) chunk by chunk - it copies chunk c as soon as
// counters[c] reports all of its rows complete - so the NVLink transfer overlaps the producer's
// compute instead of blocking its load/store pipe; the tail signals `sync` ("gradient ready").
struct PushPlan {
  const void* src[kMaxPeers];
  void* dst[kMaxPeers];
  int64_t row_bytes[kMaxPeers];
  int32_t n;
};
void launch_stream_push(const PushPlan& plan, const uint32_t* counters, int chunk_rows,
                        int64_t rows, unsigned long long timeout, int* error_flag, int blocks,
                        cudaStream_t stream, const SyncArgs& sync);
// out[i, dst_col + c] = sum_s partial[s][i, src_col + c]: requester-side sum of the W partial
// pools of multi-hot row-sliced inputs.  cols[j] = {src_col, dst_col, width}
void launch_rowslice_reduce(const float* partial, int world, int64_t rows, int64_t part_stride,
                            void* out, int64_t out_stride, int out_dtype, const int32_t* cols,
                            int n_cols, cudaStream_t stream);
// Segmented P2P pull: segs[j] = {src_rank, src_elem_off, dst_elem_off, n_elems}
void launch_gather_segments(const int64_t* segs, int n_seg, const PeerPtrs& src, void* dst,
                            int elem_bytes, int64_t max_seg_elems, cudaStream_t stream);
// Ragged P2P pull + global CSR build: segs[j] = {src_val_off, dst_item_off, splits_off, goff_off}
void launch_gather_ragged(const int64_t* segs, int n_seg, const PeerPtrs& src_vals,
                          const PeerPtrs& src_splits, void* dst_vals, int64_t* goff, int64_t b,
                          int world, int elem_bytes, int64_t max_cap, cudaStream_t stream);
// dst[i] <- (slot_flag & 1 ? src1 : src0)[i] for up to 4 segments (16-byte multiples)
void launch_select_copy(const void* const* src0, const void* const* src1, void* const* dst,
                        const int64_t* nbytes, int count, const int* slot_flag, int sm_count,
                        cudaStream_t stream);
// Copy/cast a strided 2-D block into a (symmetric) buffer: dst[r, c] = cast(src[r, c])
void launch_copy_cast_2d(const void* src, int64_t src_stride, void* dst, int64_t dst_stride,
                         int64_t rows, int64_t cols, int src_dtype, int dst_dtype, float scale,
                         cudaStream_t stream);

// ---- dense-side kernels (DLRM interaction, fused elementwise + loss + optimizer) ------------
bool launch_interact_fwd(const void* bottom, int64_t bottom_stride, const void* emb,
                         int64_t emb_stride, int n_emb, int dim, void* z, int64_t z_stride,
                         int z_width, int64_t batch, int sm_count, cudaStream_t stream,
                         const SyncArgs& sync);
// The embedding gradient goes either to one local buffer (demb, routes == nullptr) or, piece by
// piece, straight into the owners' receive buffers over NVLink (routes: columns are relative to
// the concatenated [n_emb * dim] embedding row).
// Tables the interaction backward updates itself (single-GPU SGD step): the gradient of embedding
// row f of F (bf16, as the routed copy-out would store it) is widened, scaled and reduced straight
// into table[(row_base + id) * 128 + col] when bit f of `mask` is set; the other rows go through
// the routes.  One-hot ids of feature f: ids[f][sample] + id_shift[f], valid below sub_rows[f]
// (others are skipped).  scale *= *scale_ptr when scale_ptr is set (the device learning rate).
constexpr int kMaxInteractApply = 31;
struct InteractApply {
  float* table[kMaxInteractApply];  // fused fp32 table, 128 columns, 16-byte aligned
  const void* ids[kMaxInteractApply];
  int64_t row_base[kMaxInteractApply];
  int64_t sub_rows[kMaxInteractApply];
  int64_t id_shift[kMaxInteractApply];
  const float* scale_ptr;
  float scale;
  uint32_t mask;
  int32_t ids64;
};

bool launch_interact_bwd(const void* bottom, int64_t bottom_stride, const void* emb,
                         int64_t emb_stride, int n_emb, int dim, const void* dz,
                         int64_t dz_stride, void* dbottom, int64_t dbottom_stride, void* demb,
                         int64_t demb_stride, float emb_grad_scale, int64_t batch, int sm_count,
                         cudaStream_t stream, const GradRoute* routes, int n_routes,
                         const SyncArgs& sync, uint32_t* done_counters = nullptr,
                         int chunk_rows = 0, const InteractApply* apply = nullptr);
// 1-D average pooling over bf16 rows ("same" padding; the synthetic models' interaction)
void launch_avgpool_fwd(const void* x, int64_t x_stride, int n, void* out, int64_t out_stride,
                        int out_len, int stride, int left, int64_t rows, cudaStream_t stream);
void launch_avgpool_bwd(const void* dout, int64_t dout_stride, int out_len, void* dx,
                        int64_t dx_stride, int n, int stride, int left, int64_t rows,
                        cudaStream_t stream);
void launch_relu_bwd_bias(void* dy, const void* y, float* db, int64_t rows, int cols,
                          cudaStream_t stream);
// Low-rank cross network (DLRM-DCNv2), [rows, cols] bf16 row-major, cols a multiple of 8, 16-byte
// aligned.  cross_fwd: out = x0 * s + xl over n elements.  cross_bwd: g = dy * x0,
// db[c] += sum_rows dy * x0 (fp32).  cross_dx0: d_chain + sum_l dy_l * s_l, columns below
// emb_cols into dx0, the rest into d_bottom [rows, cols - emb_cols].
constexpr int kMaxCrossLayers = 8;
struct CrossTerms {
  const void* dy[kMaxCrossLayers];
  const void* s[kMaxCrossLayers];
  int n;
};
void launch_cross_fwd(const void* x0, const void* s, const void* xl, void* out, int64_t n,
                      int sm_count, cudaStream_t stream);
void launch_cross_bwd(const void* dy, const void* x0, void* g, float* db, int64_t rows, int cols,
                      cudaStream_t stream);
void launch_cross_dx0(const void* d_chain, const CrossTerms& terms, void* dx0, void* d_bottom,
                      int64_t rows, int cols, int emb_cols, cudaStream_t stream);
bool launch_head_loss(const void* x, int K, const void* w, const void* bias, const float* labels,
                      int64_t batch, float inv_batch, void* dx, float* dw, float* db,
                      float* dbias_prev, float* loss_sum, float* logits_out, int sm_count,
                      cudaStream_t stream);
// Forward-only head for evaluation: probs = sigmoid(<x, w> + b) for every row; rows below
// *n_valid (device word) also add into hist [2, nb] (int64), loss_sum (fp64) and count (int64).
bool launch_head_eval(const void* x, int K, const void* w, const void* bias, const float* labels,
                      int64_t batch, const int64_t* n_valid, float* probs, int64_t* hist, int nb,
                      double* loss_sum, int64_t* count, int sm_count, cudaStream_t stream);
// Exact ROC AUC of the evaluation (eval_auc.cu, utils/metrics.py ExactAUC).  auc_append: rows
// below *n_valid become keys (bits(p) << 1 | label > 0.5) at keys[state[0] + i]; state (int64):
// [0] keys stored, [1] rows dropped because they would pass `capacity`, [2] rows whose p is NaN
// or outside [0, 1] (not stored), [3] block ticket, 0 between launches.
void launch_auc_append(const float* probs, const float* labels, int64_t batch,
                       const int64_t* n_valid, uint32_t* keys, int64_t capacity, int64_t* state,
                       int sm_count, cudaStream_t stream);
// auc_count: out = [P, N, U2] (int64) of n keys sorted ascending by radix_sort_keys32
size_t auc_count_temp_bytes(int64_t n);
void launch_auc_count(void* temp, const uint32_t* sorted_keys, int64_t n, int64_t* out,
                      cudaStream_t stream);
// weight_decay != 0: p32 -= lr * (grad_scale * g32 + weight_decay * p32) (both decay modes)
void launch_sgd_update(float* p32, void* p16, float* g32, const float* lr_ptr, float grad_scale,
                       int64_t n, int sm_count, cudaStream_t stream, float weight_decay = 0.f);
// Fused dense Adagrad (kind kOptAdagrad, s0 = accumulator) or Adam (kOptAdam, s0 / s1 = m / v,
// *step_ptr = t after this step) + bf16 re-cast + gradient zeroing over n (multiple of 4) fp32
// elements; false for another kind.  weight_decay with weight_decay_mode kWeightDecayL2 or
// kWeightDecayDecoupled, as the embedding update applies it.
bool launch_dense_opt(int kind, float* p32, void* p16, float* g32, float* s0, float* s1,
                      const float* lr_ptr, const float* step_ptr, float beta1, float beta2,
                      float eps, int64_t n, int sm_count, cudaStream_t stream,
                      float weight_decay = 0.f, int weight_decay_mode = kWeightDecayL2);
// Fused dense momentum SGD (torch.optim.SGD, dampening 0) with buffer b over n (multiple of 4) fp32
// elements + bf16 re-cast + gradient zeroing; the update of kOptMomentum in the embedding kernels,
// with weight_decay in either mode.
void launch_dense_momentum(float* p32, void* p16, float* g32, float* b, const float* lr_ptr,
                           float momentum, bool nesterov, int64_t n, int sm_count,
                           cudaStream_t stream, float weight_decay, int weight_decay_mode);
void launch_cast_pad(const float* src, int src_cols, void* dst, int dst_cols, int64_t rows,
                     cudaStream_t stream);

// ---- hand-written wgmma / TMA GEMM with fused bias + activation epilogue --------------------
bool launch_gemm_tn_fused(const void* A, int64_t lda, const void* B, int64_t ldb, const void* bias,
                          void* C, int64_t ldc, int M, int N, int K, int epi, const void* act,
                          int64_t ldact, float* colsum, int block_n, int sm_count,
                          cudaStream_t stream);
bool launch_gemm_tn_bias_act(const void* A, int64_t lda, const void* B, int64_t ldb,
                             const void* bias, void* C, int64_t ldc, int M, int N, int K,
                             bool relu, int block_n, int sm_count, cudaStream_t stream);

}  // namespace de
