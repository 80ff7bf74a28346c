// Row-sparse embedding bags for the CTR models (sm_90a, fp32 tables): the reference declares its embeddings
// is_sparse=True (example/ctr/ctr/save_program.py:75-144), so a step touches only the rows its batch looked up.
//
//   * forward: mean-pooled embedding bag over CSR bags (ids [nnz], offsets [B] = bag starts, nn.EmbeddingBag's
//     convention; an empty bag yields zeros) or fixed-length bags [B, L] (implicit offsets b * L);
//   * backward: the uncoalesced row-sparse gradient, one row per looked-up element k:
//         indices[k] = ids[k],   values[k, :] = dout[bag(k), :] / len(bag(k))
//     (what nn.EmbeddingBag(sparse=True) returns) -- no dense [V, D] tensor anywhere;
//   * lazy Adam over the rows of such gradients, for up to kMaxSparseTables tables of one width D in one launch: the
//     rows get the sort key table << 40 | id, the keys are stably sorted, and every run of equal keys is summed in a
//     fixed order and updates only that row's weights, m and v (Paddle's adam with lazy_mode=True, FlatAdam's formula
//     mhat / (sqrt(vhat) + eps), bias correction from a device step counter).  Rows outside the gradients are not
//     read or written.
//
// D is 10 for the embeddings and 1 for DeepFM's first-order tables, so one warp per bag with lanes over D would leave
// 22 or 31 of 32 lanes idle: the forward maps consecutive threads to (bag, column) pairs, the backward to (element,
// column) pairs, and the optimizer sums a run with 32 / D rows in flight per warp.
#include "common.cuh"
#include "kernels.h"

namespace edl {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// [begin, end) of bag b: explicit offsets (CSR) or fixed length L
EDL_DEVICE void bag_range(const int64_t* __restrict__ offsets, int64_t b, int64_t B, int64_t nnz, int L, int64_t& lo,
                          int64_t& hi) {
  if (offsets != nullptr) {
    lo = offsets[b];
    hi = b + 1 < B ? offsets[b + 1] : nnz;
  } else {
    lo = b * L;
    hi = lo + L;
  }
}

// out[b, c] = mean over the bag's elements k of table[ids[k], c]; one thread per (bag, column), elements in order
__global__ void __launch_bounds__(kThreads)
emb_bag_mean_fwd_kernel(const float* __restrict__ table, const int64_t* __restrict__ ids,
                        const int64_t* __restrict__ offsets, float* __restrict__ out, int64_t B, int64_t nnz, int L,
                        int D) {
  const int64_t total = B * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D;
    const int c = (int)(i - b * D);
    int64_t lo, hi;
    bag_range(offsets, b, B, nnz, L, lo, hi);
    float acc = 0.f;
    for (int64_t k = lo; k < hi; ++k) acc += __ldg(table + ids[k] * D + c);
    out[i] = hi > lo ? acc / (float)(hi - lo) : 0.f;
  }
}

// values[k, c] = dout[bag(k), c] / len(bag(k)), indices[k] = ids[k]; one thread per (element, column)
__global__ void __launch_bounds__(kThreads)
emb_bag_mean_bwd_kernel(const float* __restrict__ dout, const int64_t* __restrict__ ids,
                        const int64_t* __restrict__ offsets, int64_t* __restrict__ indices, float* __restrict__ values,
                        int64_t B, int64_t nnz, int L, int D) {
  const int64_t total = nnz * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i / D;
    const int c = (int)(i - k * D);
    int64_t b;
    if (offsets != nullptr) {
      // the last bag that starts at or before k (empty bags share their start with the next one)
      int64_t l = 0, r = B;
      while (r - l > 1) {
        const int64_t mid = (l + r) >> 1;
        if (offsets[mid] <= k) l = mid;
        else r = mid;
      }
      b = l;
    } else {
      b = k / L;
    }
    int64_t lo, hi;
    bag_range(offsets, b, B, nnz, L, lo, hi);
    values[i] = dout[b * D + c] / (float)(hi - lo);
    if (c == 0) indices[k] = ids[k];
  }
}

// Several slots at once (fixed-length bags ids [B, S, L], slot s looks up tabs.w[s]; the CTR models' 26 slots in one
// launch instead of 26).  Forward: one thread per (bag, slot, column); out [B, S, D].
__global__ void __launch_bounds__(kThreads)
emb_bags_mean_fwd_kernel(const int64_t* __restrict__ ids, float* __restrict__ out, int64_t B, int S, int L, int D,
                         const __grid_constant__ SlotTables tabs) {
  const int64_t total = B * S * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bs = i / D;
    const int c = (int)(i - bs * D);
    const float* __restrict__ table = tabs.w[bs % S];
    const int64_t* __restrict__ row = ids + bs * L;
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc += __ldg(table + row[l] * D + c);
    out[i] = L > 0 ? acc / (float)L : 0.f;
  }
}

// Backward of the above, slot-major so that every slot's gradient is one contiguous block: one thread per (element,
// column); indices [S, B * L], values [S, B * L, D]
__global__ void __launch_bounds__(kThreads)
emb_bags_mean_bwd_kernel(const float* __restrict__ dout, const int64_t* __restrict__ ids, int64_t* __restrict__ indices,
                         float* __restrict__ values, int64_t B, int S, int L, int D) {
  const int64_t total = B * S * L * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i / D;
    const int c = (int)(i - e * D);
    const int64_t bs = e / L;
    const int l = (int)(e - bs * L);
    const int64_t b = bs / S;
    const int s = (int)(bs - b * S);
    const int64_t o = ((int64_t)s * B + b) * L + l;
    values[o * D + c] = dout[bs * D + c] / (float)L;
    if (c == 0) indices[o] = ids[e];
  }
}

constexpr int kIdBits = 40;              // sort key = table << 40 | row id (V < 2^40)

// sort keys of the concatenated gradient rows of several tables: key = table << 40 | id; an id outside its table
// gets key -1 and is skipped by the update
__global__ void __launch_bounds__(kThreads)
sparse_adam_keys_kernel(const int64_t* __restrict__ ids, int64_t* __restrict__ keys, int64_t n,
                        const __grid_constant__ SparseTables tabs) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int t = 0;
    while (t + 1 < tabs.count && tabs.start[t + 1] <= i) ++t;
    const int64_t id = ids[i];
    keys[i] = (id >= 0 && id < tabs.rows[t]) ? (((int64_t)t << kIdBits) | id) : -1;
  }
}

// One warp per position k of the sorted keys; only the first position of a run of equal keys (one row of one table)
// does work.  The run [k, end) is found with ballots (sorted input: the matches are a prefix of every 32-wide window),
// its rows are summed in fp64 by G = 32 / min(D, 32) row groups (group q takes rows k + q, k + q + G, ...) whose partial sums
// group 0 adds in ascending q -- a fixed order, so the update is deterministic however many times an id repeats.
__global__ void __launch_bounds__(kThreads)
sparse_adam_kernel(const int64_t* __restrict__ sorted_keys, const int64_t* __restrict__ perm,
                   const float* __restrict__ values, int64_t n, int D, const __grid_constant__ SparseTables tabs,
                   const float* __restrict__ lr_p, const float* __restrict__ step_p, float beta1, float beta2,
                   float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (k >= n) return;
  const int64_t key = sorted_keys[k];
  if (key < 0 || (k > 0 && sorted_keys[k - 1] == key)) return;
  int64_t end = k + 1;
  for (;;) {
    const int64_t j = end + lane;
    const unsigned ball = __ballot_sync(0xffffffffu, j < n && sorted_keys[j] == key);
    end += __popc(ball);
    if (ball != 0xffffffffu) break;
  }
  const int t = (int)(key >> kIdBits);
  const int64_t id = key & ((1ll << kIdBits) - 1);
  float* __restrict__ w = tabs.w[t];
  float* __restrict__ m = tabs.m[t];
  float* __restrict__ v = tabs.v[t];
  const int lpr = D < 32 ? D : 32;     // lanes per row
  const int G = 32 / lpr;              // rows in flight
  const int grp = lane / lpr, col = lane - grp * lpr;
  const float lr = *lr_p, step = *step_p;
  const float bc1 = 1.f - powf(beta1, step);
  const float bc2 = 1.f - powf(beta2, step);
  for (int c0 = 0; c0 < D; c0 += lpr) {
    const int c = c0 + col;
    const bool active = grp < G && c < D;
    // fp64 partial sums: a run of 10^5 equal ids sums to within one fp32 rounding of the exact value
    double acc = 0.0;
    if (active)
      for (int64_t j = k + grp; j < end; j += G) acc += (double)values[perm[j] * D + c];
    double sum = acc;
    for (int q = 1; q < G; ++q) sum += __shfl_sync(0xffffffffu, acc, col + q * lpr);
    const float g = (float)sum;
    if (active && grp == 0) {
      const int64_t o = id * D + c;
      const float mi = fmaf(beta1, m[o], (1.f - beta1) * g);
      const float vi = fmaf(beta2, v[o], (1.f - beta2) * g * g);
      const float mhat = mi / bc1;
      const float vhat = vi / bc2;
      w[o] -= lr * mhat / (sqrtf(vhat) + eps);
      m[o] = mi;
      v[o] = vi;
    }
  }
}

inline int grid_for(int64_t n) {
  int64_t b = (n + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)kNumSMs * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

void embedding_bag_mean_fwd(const float* table, const int64_t* ids, const int64_t* offsets, float* out, int64_t B,
                            int64_t nnz, int L, int D, cudaStream_t s) {
  if (B * D == 0) return;
  emb_bag_mean_fwd_kernel<<<grid_for(B * D), kThreads, 0, s>>>(table, ids, offsets, out, B, nnz, L, D);
}

void embedding_bag_mean_bwd_sparse(const float* dout, const int64_t* ids, const int64_t* offsets, int64_t* indices,
                                   float* values, int64_t B, int64_t nnz, int L, int D, cudaStream_t s) {
  if (nnz * D == 0) return;
  emb_bag_mean_bwd_kernel<<<grid_for(nnz * D), kThreads, 0, s>>>(dout, ids, offsets, indices, values, B, nnz, L, D);
}

void embedding_bags_mean_fwd(const int64_t* ids, float* out, int64_t B, int S, int L, int D, const SlotTables& tabs,
                             cudaStream_t s) {
  if (B * S * D == 0) return;
  emb_bags_mean_fwd_kernel<<<grid_for(B * S * D), kThreads, 0, s>>>(ids, out, B, S, L, D, tabs);
}

void embedding_bags_mean_bwd_sparse(const float* dout, const int64_t* ids, int64_t* indices, float* values, int64_t B,
                                    int S, int L, int D, cudaStream_t s) {
  if (B * S * L * D == 0) return;
  emb_bags_mean_bwd_kernel<<<grid_for(B * S * L * D), kThreads, 0, s>>>(dout, ids, indices, values, B, S, L, D);
}

void sparse_adam_keys(const int64_t* ids, int64_t* keys, int64_t n, const SparseTables& tabs, cudaStream_t s) {
  if (n == 0) return;
  sparse_adam_keys_kernel<<<grid_for(n), kThreads, 0, s>>>(ids, keys, n, tabs);
}

void sparse_adam(const int64_t* sorted_keys, const int64_t* perm, const float* values, int64_t n, int D,
                 const SparseTables& tabs, const float* lr, const float* step, float beta1, float beta2, float eps,
                 cudaStream_t s) {
  if (n == 0) return;
  const int64_t grid = (n + kWarps - 1) / kWarps;
  sparse_adam_kernel<<<(unsigned)grid, kThreads, 0, s>>>(sorted_keys, perm, values, n, D, tabs, lr, step, beta1,
                                                         beta2, eps);
}

}  // namespace edl
