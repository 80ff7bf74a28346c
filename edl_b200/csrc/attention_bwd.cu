// Masked multi-head attention backward for sm_90a (padded layout, head dim 64 or 32, L <= 512): the training path of
// the Transformer student.  With S = Q K^T / 8 and P = softmax over the valid keys (head dim 64; 32 below),
//
//   dV = P^T dO,   dP = dO V^T,   dS = P o (dP - D) with D = rowsum(dO o O),   dQ = dS K / 8,   dK = dS^T Q / 8.
//
// P is recomputed from the forward's lse (attention.cu): P = exp2(S * log2(e) / 8 - lse), 0 for a masked key and for
// every key of a row without a valid key (lse = +inf), so such a row gets exactly zero gradients.  Three launches, none
// with atomics, so every result is bitwise reproducible:
//   attn_bwd_delta   one warp per token row: D[b, h, i] over the stored bf16 dO and O, fp32
//   attn_bwd_dkdv    one CTA per (64-key tile, head, sequence), four warps of 16 keys; loops over the query tiles
//   attn_bwd_dq      one CTA per (64-query tile, head, sequence), four warps of 16 queries; loops over the key tiles
// The products are mma.sync m16n8k16 bf16 -> fp32.  A warp keeps its 16 rows of the resident operand (K and V, or Q and
// dO) as A fragments in registers and builds the second product's A fragments (P^T / dS^T, or dS) from the first
// products' accumulators; the streamed tiles sit in shared memory row-major and transposed (row pitch 72 bf16, so the
// fragment loads of a warp hit 32 distinct banks).  dQ, dK and dV are stored straight from the accumulators into dqkv,
// laid out like qkv: [B * L, 3 * H * 64] with dQ | dK | dV column blocks, so the QKV projection's dgrad and weight
// gradient each take dqkv as one operand.
//
// Dropout (kDrop, the forward's attention dropout): with Z = keep * 1 / (1 - p) regenerated per element from (b, h, i, j)
// (philox.cuh; the mask does not depend on the tile order), dV = (Z o P)^T dO and dS = P o (Z o dP - D), D taken over the
// stored, dropped O as before (FlashAttention-2's identity).  A row without a valid key still gets zero gradients.
//
// Packed sequences (kVarlen, attention_varlen_bwd): qkv / dqkv [T, 3 * H * 64], O / dO [T, H * 64], sequence b in rows
// [cu_seqlens[b], cu_seqlens[b + 1]); lse and D are fp32 [H, T] at h * T + packed row (attention.cu's VarlenTrain), and
// the dropout index of (b, h, i, j) is ((b H + h) 512 + i) 512 + j.  The grid spans the longest sequence; a CTA reads its
// sequence's start and length L, exits when its tile starts at or past L, and otherwise runs the padded body with that
// L on the rows from the start: the same tiles and bounds, so no row outside the sequence is read as its data and the
// bits are those of the padded kernels at B = 1 (up to the dropout index).  A key is valid iff key < L and key_mask of
// its packed row is set.  D is the padded delta pass over T rows as one sequence (B = 1, L = T).
//
// Budgets (ptxas -v, sm_90a, 128 threads): attn_bwd_dkdv 175 registers (228 with dropout), attn_bwd_dq 134 (242),
// attn_bwd_delta 40, no spills; packed: attn_bwd_dkdv 173 registers (220 with dropout), attn_bwd_dq 136 (175), no
// spills;
// static shared memory 36.5 KB (dkdv: Q, Q^T, dO, dO^T tiles + lse / D) and 27.1 KB (dq: K, K^T, V tiles + key flags).
//
// Head dim 32 (template parameter D; the D = 64 instantiations compile to the SASS they had before it existed): the
// tiles are 64 x D (row pitch 72 kept, so fragment loads still hit 32 distinct banks) and their transposes D x 64; S and
// dP take K = D (two k16 steps), dQ / dK / dV are D / 8 accumulator tiles wide, dQ and dK are scaled by 1 / sqrt(32),
// and the delta pass leaves lanes 16..31 idle.  Budgets, no spills: attn_bwd_dkdv 131 registers (149 with dropout),
// attn_bwd_dq 101 (180), attn_bwd_delta 32; packed: attn_bwd_dkdv 132 (145), attn_bwd_dq 101 (160); static shared
// memory 27.5 KB (dkdv) and 22.6 KB (dq).
#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace edl {
namespace {

constexpr int kT = 64;        // tile rows (keys or queries)
constexpr int kP = 72;        // shared-memory row pitch in bf16
// 1 / sqrt(D) and 1 / sqrt(D) * log2(e) of head dim D (64 or 32), as the forward (attention.cu) forms them
template <int D>
constexpr float kInvSqrtD = D == 64 ? 0.125f : (float)(1.0 / 5.656854249492381);
template <int D>
constexpr float kScaleLog2 = D == 64 ? 0.125f * 1.4426950408889634f : (float)(1.4426950408889634 / 5.656854249492381);

EDL_DEVICE uint32_t pack2(float a, float b) {
  const __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&t);
}

EDL_DEVICE void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

EDL_DEVICE uint32_t lds(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }

// 64 rows x W columns of one head from a [B * L, ld] bf16 buffer (rows at or past L read as 0) into a row-major tile
// and, if t != nullptr, its transpose (W rows of 64)
template <int W>
EDL_DEVICE void load_tile(const __nv_bfloat16* __restrict__ src, int64_t ld, int r0, int L, __nv_bfloat16* s,
                          __nv_bfloat16* t) {
  static_assert(W == 64 || W == 32, "tile width 64 or 32");
  constexpr int kShift = W == 64 ? 3 : 2;                       // log2 of the 8-column chunks per row
  for (int v = threadIdx.x; v < kT * (W / 8); v += 128) {
    const int r = v >> kShift, c = (v & (W / 8 - 1)) * 8;
    bf16x8 x;
    if (r0 + r < L) x = *reinterpret_cast<const bf16x8*>(src + (int64_t)(r0 + r) * ld + c);
    else x = bf16x8{};
    *reinterpret_cast<bf16x8*>(s + r * kP + c) = x;
    if (t != nullptr) {
      const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&x);
#pragma unroll
      for (int i = 0; i < 8; ++i) t[(c + i) * kP + r] = e[i];
    }
  }
}

// A fragments of rows r0 .. r0 + 15 of a row-major tile, the K / 16 16-column k steps
template <int K>
EDL_DEVICE void load_afrag(const __nv_bfloat16* s, int r0, int g, int t, uint32_t (&a)[K / 16][4]) {
#pragma unroll
  for (int k = 0; k < K / 16; ++k) {
    a[k][0] = lds(s + (r0 + g) * kP + k * 16 + 2 * t);
    a[k][1] = lds(s + (r0 + g + 8) * kP + k * 16 + 2 * t);
    a[k][2] = lds(s + (r0 + g) * kP + k * 16 + 8 + 2 * t);
    a[k][3] = lds(s + (r0 + g + 8) * kP + k * 16 + 8 + 2 * t);
  }
}

// c[j] (16 x 8, j = 0..7) += A (16 x K) * Y^T, Y a row-major tile whose rows are the 64 output columns
template <int K>
EDL_DEVICE void mma_rows(float (&c)[8][4], const uint32_t (&a)[K / 16][4], const __nv_bfloat16* y, int g, int t) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < K / 16; ++k)
      mma16816(c[j], a[k], lds(y + (j * 8 + g) * kP + k * 16 + 2 * t), lds(y + (j * 8 + g) * kP + k * 16 + 8 + 2 * t));
}

// A fragments (bf16) of a 16 x 64 operand held as eight 16 x 8 accumulator tiles
EDL_DEVICE void acc_to_afrag(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    a[k][0] = pack2(c[2 * k][0], c[2 * k][1]);
    a[k][1] = pack2(c[2 * k][2], c[2 * k][3]);
    a[k][2] = pack2(c[2 * k + 1][0], c[2 * k + 1][1]);
    a[k][3] = pack2(c[2 * k + 1][2], c[2 * k + 1][3]);
  }
}

// rows r .. of a 16 x W accumulator (times `scale`) -> bf16 columns col0 .. of dqkv rows (rows at or past L skipped)
template <int W>
EDL_DEVICE void store_rows(const float (&c)[W / 8][4], __nv_bfloat16* __restrict__ dst, int64_t ld, int r, int L, int t,
                           float scale) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (r + 8 * h >= L) continue;
    __nv_bfloat16* row = dst + (int64_t)(r + 8 * h) * ld + 2 * t;
#pragma unroll
    for (int j = 0; j < W / 8; ++j)
      *reinterpret_cast<uint32_t*>(row + j * 8) = pack2(c[j][2 * h] * scale, c[j][2 * h + 1] * scale);
  }
}

// one warp per row, lane l holds columns 2 l, 2 l + 1 (lanes past D / 2 add 0)
template <int D = 64>
__global__ void __launch_bounds__(256)
attn_bwd_delta(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout, float* __restrict__ delta,
               int B, int L, int H) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= (int64_t)B * L) return;
  const int b = (int)(r / L), i = (int)(r % L);
  for (int h = 0; h < H; ++h) {
    const int64_t o = r * H * D + h * D + 2 * lane;
    float v = 0.f;
    if (2 * lane < D) {
      const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(out + o));
      const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dout + o));
      v = fmaf(x.x, y.x, x.y * y.y);
    }
    const float s = warp_sum(v);
    if (lane == 0) delta[((int64_t)b * H + h) * L + i] = s;
  }
}

template <bool kDrop, bool kVarlen = false, int D = 64>
__global__ void __launch_bounds__(128)
attn_bwd_dkdv(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ mask,
              const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ delta,
              __nv_bfloat16* __restrict__ dqkv, int L, int H, const PhiloxArgs drop,
              const int* __restrict__ cu_seqlens = nullptr, int T = 0) {
  __shared__ alignas(16) __nv_bfloat16 sQ[kT * kP], sQt[D * kP], sO[kT * kP], sOt[D * kP];
  __shared__ float sL[kT], sD[kT];
  const int k0 = blockIdx.x * kT, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t ldq = (int64_t)3 * H * D, ldo = (int64_t)H * D;
  int64_t r0 = (int64_t)b * L;                                  // the sequence's first row
  if constexpr (kVarlen) {
    r0 = cu_seqlens[b];
    L = cu_seqlens[b + 1] - (int)r0;
    if (k0 >= L) return;                                        // the grid spans the longest sequence
  }
  const __nv_bfloat16* base = qkv + r0 * ldq;
  // lse / D of head h and row i at sh + i; the dropout index of (i, j) is (dsh + i) dl + j
  const int64_t sh = kVarlen ? (int64_t)h * T + r0 : ((int64_t)b * H + h) * L;
  const int dl = kVarlen ? kAttnMaxLen : L;
  const uint64_t dsh = kVarlen ? ((uint64_t)b * H + h) * kAttnMaxLen : (uint64_t)sh;
  // this warp's 16 keys of K and V as A fragments (staged through the Q / dO tiles)
  load_tile<D>(base + (H + h) * D, ldq, k0, L, sQ, nullptr);
  load_tile<D>(base + (2 * H + h) * D, ldq, k0, L, sO, nullptr);
  __syncthreads();
  uint32_t kf[D / 16][4], vf[D / 16][4];
  load_afrag<D>(sQ, warp * 16, g, t, kf);
  load_afrag<D>(sO, warp * 16, g, t, vf);
  const int key0 = k0 + warp * 16 + g;
  bool kv[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int key = key0 + 8 * e;
    kv[e] = key < L && (mask == nullptr || mask[r0 + key] != 0);
  }
  float dk[D / 8][4], dv[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[j][e] = dv[j][e] = 0.f;
  [[maybe_unused]] PhiloxKey pk;
  if constexpr (kDrop) pk = philox_key(drop);

  for (int q0 = 0; q0 < L; q0 += kT) {
    __syncthreads();                                        // the previous tiles (or the K / V staging) are consumed
    load_tile<D>(base + h * D, ldq, q0, L, sQ, sQt);
    load_tile<D>(dout + r0 * ldo + h * D, ldo, q0, L, sO, sOt);
    if (threadIdx.x < kT) {
      const int q = q0 + threadIdx.x;
      sL[threadIdx.x] = q < L ? lse[sh + q] : INFINITY;
      sD[threadIdx.x] = q < L ? delta[sh + q] : 0.f;
    }
    __syncthreads();
    // keep bits of this thread's 32 elements, bit j * 4 + e of accumulator element [j][e] (formed before the
    // accumulators are live: the Philox rounds then need no registers the products hold)
    [[maybe_unused]] uint32_t km = 0;
    if constexpr (kDrop) {
#pragma unroll 1
      for (int i = 0; i < 32; ++i) {
        const int qc = (i >> 2) * 8 + 2 * t + (i & 1);
        const uint64_t n = (dsh + (q0 + qc)) * (uint64_t)dl + (key0 + 8 * ((i >> 1) & 1));
        km |= dropout_keep(pk, n) ? 1u << i : 0u;
      }
    }
    // S^T (keys x queries) and dP^T = V dO^T
    float p[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) p[j][e] = dp[j][e] = 0.f;
    mma_rows<D>(p, kf, sQ, g, t);
    mma_rows<D>(dp, vf, sO, g, t);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = j * 8 + 2 * t + (e & 1);
        const float pe = kv[e >> 1] ? exp2f(p[j][e] * kScaleLog2<D> - sL[qc]) : 0.f;
        if constexpr (kDrop) {
          const float z = (km >> (j * 4 + e)) & 1u ? pk.scale : 0.f;
          p[j][e] = pe * z;
          dp[j][e] = pe * (dp[j][e] * z - sD[qc]);
        } else {
          p[j][e] = pe;
          dp[j][e] = pe * (dp[j][e] - sD[qc]);
        }
      }
    // dV += P^T dO, dK += dS^T Q (the queries are the k dimension: B operands from the transposed tiles)
    uint32_t pa[4][4], sa[4][4];
    acc_to_afrag(p, pa);
    acc_to_afrag(dp, sa);
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat16* ro = sOt + (j * 8 + g) * kP + k * 16 + 2 * t;
        const __nv_bfloat16* rq = sQt + (j * 8 + g) * kP + k * 16 + 2 * t;
        mma16816(dv[j], pa[k], lds(ro), lds(ro + 8));
        mma16816(dk[j], sa[k], lds(rq), lds(rq + 8));
      }
  }
  __nv_bfloat16* drow = dqkv + r0 * ldq;
  store_rows<D>(dk, drow + (H + h) * D, ldq, key0, L, t, kInvSqrtD<D>);
  store_rows<D>(dv, drow + (2 * H + h) * D, ldq, key0, L, t, 1.f);
}

template <bool kDrop, bool kVarlen = false, int D = 64>
__global__ void __launch_bounds__(128)
attn_bwd_dq(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ mask,
            const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ delta,
            __nv_bfloat16* __restrict__ dqkv, int L, int H, const PhiloxArgs drop,
            const int* __restrict__ cu_seqlens = nullptr, int T = 0) {
  __shared__ alignas(16) __nv_bfloat16 sK[kT * kP], sKt[D * kP], sV[kT * kP];
  __shared__ uint8_t sM[kT];
  const int q0 = blockIdx.x * kT, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t ldq = (int64_t)3 * H * D, ldo = (int64_t)H * D;
  int64_t r0 = (int64_t)b * L;                                  // the sequence's first row
  if constexpr (kVarlen) {
    r0 = cu_seqlens[b];
    L = cu_seqlens[b + 1] - (int)r0;
    if (q0 >= L) return;                                        // the grid spans the longest sequence
  }
  const __nv_bfloat16* base = qkv + r0 * ldq;
  // lse / D of head h and row i at sh + i; the dropout index of (i, j) is (dsh + i) dl + j
  const int64_t sh = kVarlen ? (int64_t)h * T + r0 : ((int64_t)b * H + h) * L;
  const int dl = kVarlen ? kAttnMaxLen : L;
  const uint64_t dsh = kVarlen ? ((uint64_t)b * H + h) * kAttnMaxLen : (uint64_t)sh;
  // this warp's 16 queries of Q and dO as A fragments (staged through the K / V tiles)
  load_tile<D>(base + h * D, ldq, q0, L, sK, nullptr);
  load_tile<D>(dout + r0 * ldo + h * D, ldo, q0, L, sV, nullptr);
  __syncthreads();
  uint32_t qf[D / 16][4], of[D / 16][4];
  load_afrag<D>(sK, warp * 16, g, t, qf);
  load_afrag<D>(sV, warp * 16, g, t, of);
  const int qr = q0 + warp * 16 + g;
  float rl[2], rd[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int q = qr + 8 * e;
    rl[e] = q < L ? lse[sh + q] : INFINITY;
    rd[e] = q < L ? delta[sh + q] : 0.f;
  }
  float dq[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dq[j][e] = 0.f;
  [[maybe_unused]] PhiloxKey pk;
  if constexpr (kDrop) pk = philox_key(drop);

  for (int kb = 0; kb < L; kb += kT) {
    __syncthreads();
    load_tile<D>(base + (H + h) * D, ldq, kb, L, sK, sKt);
    load_tile<D>(base + (2 * H + h) * D, ldq, kb, L, sV, nullptr);
    if (threadIdx.x < kT) {
      const int key = kb + threadIdx.x;
      sM[threadIdx.x] = (key < L && (mask == nullptr || mask[r0 + key] != 0)) ? 1 : 0;
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = dp[j][e] = 0.f;
    mma_rows<D>(s, qf, sK, g, t);
    mma_rows<D>(dp, of, sV, g, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      [[maybe_unused]] uint32_t keep[2];
      if constexpr (kDrop) {
#pragma unroll
        for (int r = 0; r < 2; ++r)
          keep[r] = dropout_keep2(pk, (dsh + (qr + 8 * r)) * (uint64_t)dl + (kb + j * 8 + 2 * t));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = j * 8 + 2 * t + (e & 1);
        const float pe = sM[kc] ? exp2f(s[j][e] * kScaleLog2<D> - rl[e >> 1]) : 0.f;
        if constexpr (kDrop) {
          const float z = (keep[e >> 1] >> (e & 1)) & 1u ? pk.scale : 0.f;
          s[j][e] = pe * (dp[j][e] * z - rd[e >> 1]);
        } else {
          s[j][e] = pe * (dp[j][e] - rd[e >> 1]);
        }
      }
    }
    uint32_t sa[4][4];
    acc_to_afrag(s, sa);
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat16* rk = sKt + (j * 8 + g) * kP + k * 16 + 2 * t;
        mma16816(dq[j], sa[k], lds(rk), lds(rk + 8));
      }
  }
  store_rows<D>(dq, dqkv + r0 * ldq + h * D, ldq, qr, L, t, kInvSqrtD<D>);
}

template <int D>
const char* attention_bwd_d(const void* qkv, const uint8_t* mask, const void* out, const float* lse, const void* dout,
                            void* dqkv, float* delta, int B, int L, int H, cudaStream_t stream, const PhiloxArgs* drop) {
  const auto* q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  const auto* o = reinterpret_cast<const __nv_bfloat16*>(out);
  const auto* d = reinterpret_cast<const __nv_bfloat16*>(dout);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  const int64_t rows = (int64_t)B * L;
  attn_bwd_delta<D><<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(o, d, delta, B, L, H);
  const dim3 grid((L + kT - 1) / kT, H, B);
  if (drop != nullptr) {
    attn_bwd_dkdv<true, false, D><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, *drop);
    attn_bwd_dq<true, false, D><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, *drop);
  } else {
    attn_bwd_dkdv<false, false, D><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, PhiloxArgs{});
    attn_bwd_dq<false, false, D><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, PhiloxArgs{});
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

template <int D>
const char* attention_varlen_bwd_d(const void* qkv, const int* cu_seqlens, const uint8_t* key_mask, const void* out,
                                   const float* lse, const void* dout, void* dqkv, float* delta, int T, int B,
                                   int max_len, int H, cudaStream_t stream, const PhiloxArgs* drop) {
  const auto* q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  const auto* o = reinterpret_cast<const __nv_bfloat16*>(out);
  const auto* d = reinterpret_cast<const __nv_bfloat16*>(dout);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  attn_bwd_delta<D><<<(unsigned)(((int64_t)T + 7) / 8), 256, 0, stream>>>(o, d, delta, 1, T, H);   // D [H, T]
  const dim3 grid((max_len + kT - 1) / kT, H, B);
  if (drop != nullptr) {
    attn_bwd_dkdv<true, true, D><<<grid, 128, 0, stream>>>(q, key_mask, d, lse, delta, dq, max_len, H, *drop,
                                                            cu_seqlens, T);
    attn_bwd_dq<true, true, D><<<grid, 128, 0, stream>>>(q, key_mask, d, lse, delta, dq, max_len, H, *drop,
                                                          cu_seqlens, T);
  } else {
    attn_bwd_dkdv<false, true, D><<<grid, 128, 0, stream>>>(q, key_mask, d, lse, delta, dq, max_len, H, PhiloxArgs{},
                                                             cu_seqlens, T);
    attn_bwd_dq<false, true, D><<<grid, 128, 0, stream>>>(q, key_mask, d, lse, delta, dq, max_len, H, PhiloxArgs{},
                                                           cu_seqlens, T);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

const char* attention_bwd(const void* qkv, const uint8_t* mask, const void* out, const float* lse, const void* dout,
                          void* dqkv, float* delta, int B, int L, int H, int D, cudaStream_t stream,
                          const PhiloxArgs* drop) {
  if (!attention_supported(B, L, H, D)) return "attention_bwd: unsupported shape (head dim 32 or 64, 1 <= L <= 512)";
  return D == 64 ? attention_bwd_d<64>(qkv, mask, out, lse, dout, dqkv, delta, B, L, H, stream, drop)
                 : attention_bwd_d<32>(qkv, mask, out, lse, dout, dqkv, delta, B, L, H, stream, drop);
}

const char* attention_varlen_bwd(const void* qkv, const int* cu_seqlens, const uint8_t* key_mask, const void* out,
                                 const float* lse, const void* dout, void* dqkv, float* delta, int T, int B, int max_len,
                                 int H, int D, cudaStream_t stream, const PhiloxArgs* drop) {
  if (!attention_varlen_supported(T, B, max_len, H, D))
    return "attention_varlen_bwd: unsupported shape (head dim 32 or 64, T >= 1, 1 <= max_len <= 512)";
  return D == 64 ? attention_varlen_bwd_d<64>(qkv, cu_seqlens, key_mask, out, lse, dout, dqkv, delta, T, B, max_len, H,
                                              stream, drop)
                 : attention_varlen_bwd_d<32>(qkv, cu_seqlens, key_mask, out, lse, dout, dqkv, delta, T, B, max_len, H,
                                              stream, drop);
}

}  // namespace edl
