// COO -> CSR conversion and the IntegerLookup hash table for sm_90a.
//
// IntegerLookup maps raw int64 keys to contiguous indices [1, capacity) on the fly; index 0 is the
// out-of-vocabulary bucket once the vocabulary is full.  The table is open addressed with linear
// probing over 16-byte (key, value) slots: a writer claims a slot by CAS on the key word, draws
// the next free index from a single device counter (no O(capacity) scan for free indices, cf.
// reference cc/kernels/embedding_lookup_kernels.cu:395-405) and then publishes the value with a
// release store; readers that hit a claimed-but-unpublished slot spin on an acquire load.
//
// Capability parity: RowToSplit (embedding_lookup_kernels.cu:337-376), SearchAndUpdate +
// cuco::static_map insert_and_find/find + initialize (:383-516).
#include "common.cuh"

namespace de {

namespace {

constexpr int64_t kEmptyKey = -1;
constexpr int64_t kUnpublished = -1;

// row_splits[r] = first COO entry whose row index is >= r (entries sorted by row)
__global__ void row_to_split_kernel(const int64_t* __restrict__ coo, int64_t nnz, int64_t num_rows,
                                    int64_t* __restrict__ splits) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r > num_rows) return;
  int64_t lo = 0, hi = nnz;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (coo[2 * mid] < r) lo = mid + 1;
    else hi = mid;
  }
  splits[r] = lo;
}

__global__ void hash_init_kernel(int64_t* table, int64_t n_slots) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < 2 * n_slots) table[i] = -1;
}

// 64-bit finalizer of MurmurHash3 (fmix64): good avalanche for sequential / hashed-hex keys
__device__ __forceinline__ uint64_t mix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return k;
}

__device__ __forceinline__ int64_t ld_acquire_i64(const int64_t* p) {
  int64_t v;
  asm volatile("ld.acquire.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_i64(int64_t* p, int64_t v) {
  asm volatile("st.release.gpu.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__global__ void integer_lookup_kernel(int64_t* __restrict__ table, int64_t n_slots,
                                      uint32_t* __restrict__ counts,
                                      int64_t* __restrict__ next_index,
                                      const int64_t* __restrict__ keys, int64_t n, int64_t capacity,
                                      int64_t* __restrict__ out) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (tid >= n) return;
  const int64_t key = keys[tid];
  int64_t value = 0;
  if (key != kEmptyKey) {
    int64_t slot = static_cast<int64_t>(mix64(static_cast<uint64_t>(key)) %
                                        static_cast<uint64_t>(n_slots));
    for (int64_t probe = 0; probe < n_slots; ++probe) {
      int64_t* kp = table + 2 * slot;
      int64_t cur = ld_acquire_i64(kp);
      if (cur == kEmptyKey) {
        // vocabulary exhausted: look-ups only, so the table never fills up with OOV keys
        if (ld_acquire_i64(next_index) >= capacity) {
          value = 0;
          break;
        }
        const unsigned long long prev =
            atomicCAS(reinterpret_cast<unsigned long long*>(kp),
                      static_cast<unsigned long long>(kEmptyKey),
                      static_cast<unsigned long long>(key));
        cur = static_cast<int64_t>(prev);
        if (cur == kEmptyKey) {  // slot claimed by this thread: allocate the index, publish it
          // Threads that raced past the capacity check above may find the counter exhausted:
          // their key is recorded as OOV (value 0).  That is the contract - once the vocabulary
          // is full every new key is OOV for good (reference CU:445-464) - and it costs at most
          // one slot per thread of the launch that crossed the limit (the table has 50 % slack
          // and later launches stop inserting at the check above).
          const int64_t idx = static_cast<int64_t>(
              atomicAdd(reinterpret_cast<unsigned long long*>(next_index), 1ULL));
          value = idx < capacity ? idx : 0;
          st_release_i64(kp + 1, value);
          break;
        }
      }
      if (cur == key) {  // present (maybe still being published by its owner)
        // the owner is a few instructions away from its release store; like every other wait of
        // this code base the spin is bounded (a lost publisher yields OOV, not a hung GPU)
        int64_t v = ld_acquire_i64(kp + 1);
        for (int spin = 0; v == kUnpublished && spin < (1 << 22); ++spin) {
          __nanosleep(32);
          v = ld_acquire_i64(kp + 1);
        }
        value = v == kUnpublished ? 0 : v;
        break;
      }
      slot = slot + 1 == n_slots ? 0 : slot + 1;
    }
  }
  atomicAdd(counts + value, 1u);
  out[tid] = value;
}

}  // namespace

void launch_row_to_split(const int64_t* coo_indices, int64_t nnz, int64_t num_rows,
                         int64_t* row_splits, cudaStream_t stream) {
  const int threads = 256;
  const int64_t blocks = (num_rows + 1 + threads - 1) / threads;
  row_to_split_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(coo_indices, nnz,
                                                                             num_rows, row_splits);
}

void launch_hash_init(int64_t* table, int64_t n_slots, cudaStream_t stream) {
  const int threads = 256;
  const int64_t blocks = (2 * n_slots + threads - 1) / threads;
  hash_init_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(table, n_slots);
}

void launch_integer_lookup(int64_t* table, int64_t n_slots, uint32_t* counts, int64_t* next_index,
                           const int64_t* keys, int64_t n, int64_t capacity, int64_t* out,
                           cudaStream_t stream) {
  if (n <= 0) return;
  const int threads = 256;
  const int64_t blocks = (n + threads - 1) / threads;
  integer_lookup_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
      table, n_slots, counts, next_index, keys, n, capacity, out);
}

}  // namespace de
