// Masked multi-head attention forward for sm_90a (the ERNIE / BERT encoder of the NLP teacher and of the Transformer
// student).
//
//   O[b, i, h, :] = sum_j softmax_j(Q[b, i, h, :] . K[b, j, h, :] / 8 + mask[b, j]) V[b, j, h, :],   head dim 64
//
// Q, K and V are read in place from the QKV projection's output [B * L, 3 * H * 64] (columns [0, H*64) are Q, then K,
// then V) through ONE 4-D tensor map {64, 3H, L, B}: head h of Q / K / V is coordinate h / H + h / 2H of dimension 1.
// O is written as [B * L, H * 64], the output projection's input.  mask is uint8 [B, L], 1 = attend; any pattern.
//
// One CTA per (128-query tile, head, sequence):
//   warp 0        TMA producer: the Q tile once, then 64-key K / V tiles through a kStages mbarrier ring
//   warps 4..11   two consumer warpgroups of 64 query rows each:
//                 S = Q K^T (four wgmma m64n64k16, both operands K-major) -> fp32 registers, masked keys -> -inf,
//                 online softmax in the fragment registers (exp2 with log2(e) / 8 folded into the scale),
//                 P packed to bf16 in registers, O += P V (register-A wgmma, V MN-major),
//                 O / rowsum -> bf16 -> swizzled staging (the group's own half of the Q tile) -> TMA store.
// Rows and keys at or past L are zero-filled by the TMA loads, masked as keys and clipped by the TMA store.  A row
// sum is taken over the bf16-ROUNDED probabilities that enter P V, so O is a convex combination of V rows up to fp32
// accumulation; a query row without any valid key stores 0.
//
// Variable-length batches (attention_varlen_fwd): sequences packed back to back, qkv [T, 3 * H * 64], sequence b in rows
// [cu_seqlens[b], cu_seqlens[b + 1]).  The rows after a sequence are the next sequence's tokens, so one map over the
// whole buffer would neither zero-fill nor clip at its end.  A prologue kernel therefore writes each sequence its own
// pair of maps (tensormap.replace of the global address and the row count of a template map, published with
// tensormap.cp_fenceproxy); the attention kernel acquires them and runs the same body with L = len_b.  A sequence's
// output thus depends on its own rows only, whatever the others hold (NaN included), and nothing is stored outside it.
//
// Training: with lse != nullptr the padded kernel also stores, per (b, h, query), lse = m + log2(l) in the log2 units of
// the scaled scores (m the row max of S / 8 * log2(e), l the row sum over the bf16-rounded probabilities), or +inf for a
// row without a valid key; attention_bwd.cu recomputes P = exp2(S / 8 * log2(e) - lse) from it.  The store sits after O
// is formed, so O does not depend on whether lse is given.  The packed layout's training instantiation (Seq =
// VarlenTrain, a separate type, so the inference kernel the teacher serves with is not touched) stores the same lse in
// fp32 [H, T] at h * T + packed row: the 64 queries of a consumer group are contiguous.
//
// Budgets (ptxas -v, sm_90a, __launch_bounds__(384, 1)): padded 98 registers (167 with dropout), packed inference 98,
// packed training 101 (164 with dropout), no spills.
//
// Dropout on the attention probabilities (training instantiations, kDrop): element (b, h, i, j) of P has the flat index
// ((b H + h) L + i) L + j in the mask of philox.cuh in the padded layout, and ((b H + h) 512 + i) 512 + j in the packed
// one (the fixed stride kAttnMaxLen keeps the index ranges of the sequences disjoint whatever their lengths).  A dropped
// probability is zeroed in the bf16 A fragment after the row sum has taken it, so m, l and lse stay those of the
// undropped softmax (lse is bitwise the p = 0 lse) and the scale 1 / (1 - p) is applied to the fp32 output together
// with 1 / l.
#include <cuda.h>

#include <type_traits>

#include "gemm.h"
#include "kernels.h"
#include "philox.cuh"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kAttnThreads = 384;
constexpr int kAttnStages = 3;
constexpr int kHalfBytes = 64 * 128;                            // 64 rows of 64 bf16
constexpr int kQBytes = 2 * kHalfBytes;
constexpr int kKVBytes = 2 * kHalfBytes;                        // K tile, then V tile
constexpr int kMaskOffset = kQBytes + kAttnStages * kKVBytes;
constexpr int kBarOffset = kMaskOffset + kAttnMaxLen;
constexpr int kAttnSmem = kBarOffset + 128 + 1024;              // barriers + alignment slack
constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;      // 1 / sqrt(64) * log2(e)

EDL_DEVICE uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&t);
}

EDL_DEVICE void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(ptx::smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

EDL_DEVICE void acquire_tmap(const CUtensorMap* m) {
  asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// Sequence layout of a packed batch: offsets [B + 1] and the per-sequence maps [B][Q/K/V, O] of the prologue.
struct Varlen {
  const int* cu_seqlens;
  const CUtensorMap* maps;
};

// The packed layout in training: also stores lse [H, T] (T packed rows), and may drop probabilities
struct VarlenTrain {
  const int* cu_seqlens;
  const CUtensorMap* maps;
  int T;
};

// Seq = int: the padded layout, seq = L for every sequence (tmQKV / tmO span the whole batch).  Seq = Varlen: packed,
// inference.  Seq = VarlenTrain: packed, training.  kDrop: dropout on P with the mask of `drop` (training only).
template <typename Seq, bool kDrop = false>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO,
                     const uint8_t* __restrict__ mask, Seq seq, int H, float* __restrict__ lse, const PhiloxArgs drop) {
  constexpr bool kVarlenTrain = std::is_same<Seq, VarlenTrain>::value;
  constexpr bool kVarlen = std::is_same<Seq, Varlen>::value || kVarlenTrain;
  static_assert(!(kVarlen && kDrop) || kVarlenTrain, "dropout: training instantiations only");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sq = smem;
  uint8_t* smask = smem + kMaskOffset;
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(smem + kBarOffset);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kAttnStages;

  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  int L, bc;                                                     // sequence length, batch coordinate in the maps
  int64_t start;                                                 // first row of a packed sequence
  const CUtensorMap* mQKV = &tmQKV;
  const CUtensorMap* mO = &tmO;
  if constexpr (kVarlen) {
    start = seq.cu_seqlens[b];
    L = seq.cu_seqlens[b + 1] - seq.cu_seqlens[b];
    if (q0 >= L) return;                                         // the grid spans the longest sequence
    mQKV = seq.maps + 2 * b;
    mO = mQKV + 1;
    bc = 0;
  } else {
    L = seq;
    start = 0;                                                   // (b * L, formed at its use)
    bc = b;
  }
  const int groups = L - q0 > 64 ? 2 : 1;                       // consumer groups with at least one query row < L
  const int n_kt = (L + 63) / 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    if constexpr (kVarlen) {
      acquire_tmap(mQKV);
      acquire_tmap(mO);
    }
    ptx::prefetch_tmap(mQKV);
    ptx::prefetch_tmap(mO);
    ptx::mbar_init(q_bar, 1);
    for (int s = 0; s < kAttnStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], groups);
    }
    ptx::fence_barrier_init();
  }
  // key validity of the whole row, padded to whole key tiles: keys at or past L are never attended
  for (int j = threadIdx.x; j < n_kt * 64; j += kAttnThreads)
    smask[j] = (j < L && (mask == nullptr || mask[kVarlen ? start + j : (int64_t)b * L + j] != 0)) ? 1 : 0;
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------ TMA producer (whole warp loops, one lane issues)
    if (ptx::elect_one()) {
      ptx::mbar_arrive_expect_tx(q_bar, groups * kHalfBytes);
      for (int g = 0; g < groups; ++g) ptx::tma_load_4d(sq + g * kHalfBytes, mQKV, q_bar, 0, h, q0 + g * 64, bc);
    }
    __syncwarp();
    for (int kt = 0; kt < n_kt; ++kt) {
      const int s = kt % kAttnStages;
      ptx::mbar_wait(&empty_bar[s], ((kt / kAttnStages) & 1) ^ 1);
      uint8_t* sk = smem + kQBytes + s * kKVBytes;
      if (ptx::elect_one()) {
        ptx::mbar_arrive_expect_tx(&full_bar[s], kKVBytes);
        ptx::tma_load_4d(sk, mQKV, &full_bar[s], 0, H + h, kt * 64, bc);
        ptx::tma_load_4d(sk + kHalfBytes, mQKV, &full_bar[s], 0, 2 * H + h, kt * 64, bc);
      }
      __syncwarp();
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------ consumers: 64 query rows per warpgroup
    const int cw = (warp - 4) >> 2;
    if (cw >= groups) return;                                   // every row of this half is past L
    const int row = (warp & 3) * 16 + (lane >> 2);              // first fragment row (the second: + 8)
    const int cq = (lane & 3) * 2;
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};      // running max (scaled, log2 units) and row sum
    [[maybe_unused]] PhiloxKey pk;
    [[maybe_unused]] uint64_t nrow[2];                          // flat mask index of key 0 of this thread's two rows
    if constexpr (kDrop) {
      pk = philox_key(drop);
      const int dl = kVarlen ? kAttnMaxLen : L;                  // the mask's row stride: L padded, 512 packed
#pragma unroll
      for (int r = 0; r < 2; ++r) nrow[r] = (((uint64_t)b * H + h) * dl + (q0 + cw * 64 + row + 8 * r)) * (uint64_t)dl;
    }
    ptx::mbar_wait(q_bar, 0);
    const uint64_t dq = ptx::make_smem_desc(ptx::smem_u32(sq + cw * kHalfBytes), 16, 1024);
    for (int kt = 0; kt < n_kt; ++kt) {
      const int s = kt % kAttnStages;
      ptx::mbar_wait(&full_bar[s], (kt / kAttnStages) & 1);
      const uint32_t sk = ptx::smem_u32(smem + kQBytes + s * kKVBytes);
      const uint64_t dk = ptx::make_smem_desc(sk, 16, 1024);
      const uint64_t dv = ptx::make_smem_desc(sk + kHalfBytes, 8192, 1024);
      float sc[32];
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::WgmmaBf16<64, 0, 0>::mma(sc, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k != 0 ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      // scale + mask, row maxima (a row's 64 columns live in the four lanes of a quad)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kt * 64 + j * 8 + cq;
        const bool v0 = smask[key] != 0, v1 = smask[key + 1] != 0;
        sc[4 * j] = v0 ? sc[4 * j] * kScaleLog2 : -INFINITY;
        sc[4 * j + 1] = v1 ? sc[4 * j + 1] * kScaleLog2 : -INFINITY;
        sc[4 * j + 2] = v0 ? sc[4 * j + 2] * kScaleLog2 : -INFINITY;
        sc[4 * j + 3] = v1 ? sc[4 * j + 3] * kScaleLog2 : -INFINITY;
        mx[0] = fmaxf(mx[0], fmaxf(sc[4 * j], sc[4 * j + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
      }
      float base[2], alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m[r], mx[r]);
        // no valid key so far: nothing has been accumulated, keep everything at 0 (no inf - inf)
        alpha[r] = mn == -INFINITY ? 1.f : exp2f(m[r] - mn);
        base[r] = mn == -INFINITY ? 0.f : mn;
        m[r] = mn;
      }
      // probabilities -> bf16 A fragments; the row sums take the rounded values that P V uses
      uint32_t pa[4][4];
      float ls[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t lo = pack_bf16(exp2f(sc[4 * j] - base[0]), exp2f(sc[4 * j + 1] - base[0]));
        uint32_t hi = pack_bf16(exp2f(sc[4 * j + 2] - base[1]), exp2f(sc[4 * j + 3] - base[1]));
        const float2 flo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lo));
        const float2 fhi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hi));
        ls[0] += flo.x + flo.y;
        ls[1] += fhi.x + fhi.y;
        if constexpr (kDrop) {
          const int key = kt * 64 + j * 8 + cq;
          const uint32_t k0 = dropout_keep2(pk, nrow[0] + key), k1 = dropout_keep2(pk, nrow[1] + key);
          lo &= ((k0 & 1u) ? 0xFFFFu : 0u) | ((k0 & 2u) ? 0xFFFF0000u : 0u);
          hi &= ((k1 & 1u) ? 0xFFFFu : 0u) | ((k1 & 2u) ? 0xFFFF0000u : 0u);
        }
        pa[j >> 1][(j & 1) * 2] = lo;
        pa[j >> 1][(j & 1) * 2 + 1] = hi;
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + ls[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
        o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
      }
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::WgmmaBf16RegA64<1>::mma(o, pa[k], dv + (uint64_t)(128 * k), 1u);   // 16 V rows = 2 KB
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[s]);
    }
    // ---- epilogue: O / rowsum -> bf16 -> this group's half of the Q tile (no longer read) -> TMA store (clipped at L)
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
      inv[r] = l[r] > 0.f ? (kDrop ? drop.scale / l[r] : 1.f / l[r]) : 0.f;
    }
    if (!kVarlen && lse != nullptr && (lane & 3) == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int qi = q0 + cw * 64 + row + 8 * r;
        if (qi < L) lse[((int64_t)b * H + h) * L + qi] = l[r] > 0.f ? m[r] + log2f(l[r]) : INFINITY;
      }
    }
    if constexpr (kVarlenTrain) {
      if ((lane & 3) == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qi = q0 + cw * 64 + row + 8 * r;
          if (qi < L) lse[(int64_t)h * seq.T + start + qi] = l[r] > 0.f ? m[r] + log2f(l[r]) : INFINITY;
        }
      }
    }
    uint8_t* st = sq + cw * kHalfBytes;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(st + row * 128 + ((j ^ (row & 7)) << 4) + cq * 2) =
          pack_bf16(o[4 * j] * inv[0], o[4 * j + 1] * inv[0]);
      *reinterpret_cast<uint32_t*>(st + (row + 8) * 128 + ((j ^ ((row + 8) & 7)) << 4) + cq * 2) =
          pack_bf16(o[4 * j + 2] * inv[1], o[4 * j + 3] * inv[1]);
    }
    ptx::fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
    if ((threadIdx.x & 127) == 0) {
      if constexpr (kVarlen) acquire_tmap(mO);
      tma_store_4d(mO, st, 0, h, q0 + cw * 64, bc);
      ptx::tma_store_commit();
      ptx::tma_store_wait_read0();
    }
  }
}

// One warp per sequence: copy the template maps to shared memory, point them at the sequence's first row, set their
// row count to its length, and publish them to maps[2 b], maps[2 b + 1] for the tensor-map proxy.
__global__ void __launch_bounds__(128)
attention_varlen_maps_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO,
                             const void* qkv, void* out, const int* __restrict__ cu_seqlens, CUtensorMap* maps, int B,
                             int H) {
  __shared__ alignas(128) CUtensorMap sm[4][2];
  const int w = threadIdx.x >> 5, b = blockIdx.x * 4 + w;
  if (b >= B) return;                                           // whole warps
  CUtensorMap* s = sm[w];
  if ((threadIdx.x & 31) == 0) {
    const int start = cu_seqlens[b];
    const int len = max(cu_seqlens[b + 1] - start, 1);          // a sequence with len < 1 launches no work
    s[0] = tmQKV;
    s[1] = tmO;
    const uint64_t a0 = reinterpret_cast<uint64_t>(qkv) + (uint64_t)start * 3 * H * 128;
    const uint64_t a1 = reinterpret_cast<uint64_t>(out) + (uint64_t)start * H * 128;
    asm volatile("tensormap.replace.tile.global_address.shared::cta.b1024.b64 [%0], %1;" ::"r"(ptx::smem_u32(s)),
                 "l"(a0) : "memory");
    asm volatile("tensormap.replace.tile.global_address.shared::cta.b1024.b64 [%0], %1;" ::"r"(ptx::smem_u32(s + 1)),
                 "l"(a1) : "memory");
    asm volatile("tensormap.replace.tile.global_dim.shared::cta.b1024.b32 [%0], 2, %1;" ::"r"(ptx::smem_u32(s)),
                 "r"(len) : "memory");
    asm volatile("tensormap.replace.tile.global_dim.shared::cta.b1024.b32 [%0], 2, %1;" ::"r"(ptx::smem_u32(s + 1)),
                 "r"(len) : "memory");
  }
  __syncwarp();
  for (int i = 0; i < 2; ++i)
    asm volatile("tensormap.cp_fenceproxy.global.shared::cta.tensormap::generic.release.gpu.sync.aligned [%0], [%1], 128;"
                 ::"l"(reinterpret_cast<uint64_t>(maps + 2 * b + i)), "r"(ptx::smem_u32(s + i)) : "memory");
}

template <typename Seq, bool kDrop = false>
const char* launch_attention(const CUtensorMap& tmQKV, const CUtensorMap& tmO, const uint8_t* mask, Seq seq, int H,
                             dim3 grid, cudaStream_t stream, float* lse = nullptr, const PhiloxArgs& drop = PhiloxArgs{}) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_fwd_kernel<Seq, kDrop>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kAttnSmem);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    attr_set = true;
  }
  attention_fwd_kernel<Seq, kDrop><<<grid, kAttnThreads, kAttnSmem, stream>>>(tmQKV, tmO, mask, seq, H, lse, drop);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// Q / K / V and O maps {64, 3H | H, rows, batch} of a [batch * rows, 3 * H * 64] / [batch * rows, H * 64] layout
const char* encode_attention_maps(CUtensorMap* tmQKV, CUtensorMap* tmO, const void* qkv, void* out, int rows, int batch,
                                  int H) {
  const uint32_t box[4] = {64, 1, 64, 1};
  {
    const uint64_t dims[4] = {64, (uint64_t)3 * H, (uint64_t)rows, (uint64_t)batch};
    const uint64_t st[3] = {128, (uint64_t)3 * H * 128, (uint64_t)rows * 3 * H * 128};
    if (const char* e = encode_tmap_bf16(tmQKV, qkv, 4, dims, st, box)) return e;
  }
  const uint64_t dims[4] = {64, (uint64_t)H, (uint64_t)rows, (uint64_t)batch};
  const uint64_t st[3] = {128, (uint64_t)H * 128, (uint64_t)rows * H * 128};
  return encode_tmap_bf16(tmO, out, 4, dims, st, box);
}

}  // namespace

bool attention_supported(int B, int L, int H, int head_dim) {
  return B >= 1 && B <= 65535 && L >= 1 && L <= kAttnMaxLen && H >= 1 && H <= 65535 && head_dim == 64;
}

const char* attention_fwd(const void* qkv, const uint8_t* mask, void* out, int B, int L, int H, cudaStream_t stream,
                          float* lse, const PhiloxArgs* drop) {
  if (!attention_supported(B, L, H, 64)) return "attention_fwd: unsupported shape (head dim 64, 1 <= L <= 512)";
  if (drop != nullptr && lse == nullptr) return "attention_fwd: dropout is a training feature (give lse)";
  alignas(64) CUtensorMap tmQKV, tmO;
  if (const char* e = encode_attention_maps(&tmQKV, &tmO, qkv, out, L, B, H)) return e;
  const dim3 grid((L + 127) / 128, H, B);
  if (drop != nullptr) return launch_attention<int, true>(tmQKV, tmO, mask, L, H, grid, stream, lse, *drop);
  return launch_attention<int>(tmQKV, tmO, mask, L, H, grid, stream, lse);
}

bool attention_varlen_supported(int T, int B, int max_len, int H, int head_dim) {
  return T >= 1 && attention_supported(B, max_len, H, head_dim);
}

const char* attention_varlen_fwd(const void* qkv, const int* cu_seqlens, const uint8_t* key_mask, void* out, void* maps,
                                 int T, int B, int max_len, int H, cudaStream_t stream, float* lse,
                                 const PhiloxArgs* drop) {
  if (!attention_varlen_supported(T, B, max_len, H, 64))
    return "attention_varlen_fwd: unsupported shape (head dim 64, T >= 1, 1 <= max_len <= 512)";
  if (drop != nullptr && lse == nullptr) return "attention_varlen_fwd: dropout is a training feature (give lse)";
  // templates over the whole buffer; the prologue replaces the address and the row count per sequence
  alignas(64) CUtensorMap tmQKV, tmO;
  if (const char* e = encode_attention_maps(&tmQKV, &tmO, qkv, out, T, 1, H)) return e;
  CUtensorMap* m = static_cast<CUtensorMap*>(maps);
  attention_varlen_maps_kernel<<<(B + 3) / 4, 128, 0, stream>>>(tmQKV, tmO, qkv, out, cu_seqlens, m, B, H);
  if (cudaError_t e = cudaGetLastError(); e != cudaSuccess) return cudaGetErrorString(e);
  const dim3 grid((max_len + 127) / 128, H, B);
  if (lse != nullptr) {
    const VarlenTrain seq{cu_seqlens, m, T};
    if (drop != nullptr) return launch_attention<VarlenTrain, true>(tmQKV, tmO, key_mask, seq, H, grid, stream, lse, *drop);
    return launch_attention<VarlenTrain>(tmQKV, tmO, key_mask, seq, H, grid, stream, lse);
  }
  return launch_attention<Varlen>(tmQKV, tmO, key_mask, Varlen{cu_seqlens, m}, H, grid, stream);
}

}  // namespace edl
