// Masked multi-head attention backward for sm_90a (padded layout, head dim 64, L <= 512): the training path of the
// Transformer student.  With S = Q K^T / 8 and P = softmax over the valid keys,
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
// Budgets (ptxas -v, sm_90a, 128 threads): attn_bwd_dkdv 175 registers (228 with dropout), attn_bwd_dq 134 (242),
// attn_bwd_delta 40, no spills;
// static shared memory 36.5 KB (dkdv: Q, Q^T, dO, dO^T tiles + lse / D) and 27.1 KB (dq: K, K^T, V tiles + key flags).
#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace edl {
namespace {

constexpr int kT = 64;        // tile rows (keys or queries)
constexpr int kP = 72;        // shared-memory row pitch in bf16
constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;

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

// 64 rows x 64 columns of one head from a [B * L, ld] bf16 buffer (rows at or past L read as 0) into a row-major tile
// and, if t != nullptr, its transpose
EDL_DEVICE void load_tile(const __nv_bfloat16* __restrict__ src, int64_t ld, int r0, int L, __nv_bfloat16* s,
                          __nv_bfloat16* t) {
  for (int v = threadIdx.x; v < kT * 8; v += 128) {
    const int r = v >> 3, c = (v & 7) * 8;
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

// A fragments of rows r0 .. r0 + 15 of a row-major tile, the four 16-column k steps
EDL_DEVICE void load_afrag(const __nv_bfloat16* s, int r0, int g, int t, uint32_t (&a)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    a[k][0] = lds(s + (r0 + g) * kP + k * 16 + 2 * t);
    a[k][1] = lds(s + (r0 + g + 8) * kP + k * 16 + 2 * t);
    a[k][2] = lds(s + (r0 + g) * kP + k * 16 + 8 + 2 * t);
    a[k][3] = lds(s + (r0 + g + 8) * kP + k * 16 + 8 + 2 * t);
  }
}

// c[j] (16 x 8, j = 0..7) += A (16 x 64) * Y^T, Y a row-major tile whose rows are the 64 output columns
EDL_DEVICE void mma_rows(float (&c)[8][4], const uint32_t (&a)[4][4], const __nv_bfloat16* y, int g, int t) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k)
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

// rows r .. of a 16 x 64 accumulator (times `scale`) -> bf16 columns col0 .. of dqkv rows (rows at or past L skipped)
EDL_DEVICE void store_rows(const float (&c)[8][4], __nv_bfloat16* __restrict__ dst, int64_t ld, int r, int L, int t,
                           float scale) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (r + 8 * h >= L) continue;
    __nv_bfloat16* row = dst + (int64_t)(r + 8 * h) * ld + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(row + j * 8) = pack2(c[j][2 * h] * scale, c[j][2 * h + 1] * scale);
  }
}

__global__ void __launch_bounds__(256)
attn_bwd_delta(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout, float* __restrict__ delta,
               int B, int L, int H) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= (int64_t)B * L) return;
  const int b = (int)(r / L), i = (int)(r % L);
  for (int h = 0; h < H; ++h) {
    const int64_t o = r * H * 64 + h * 64 + 2 * lane;
    const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(out + o));
    const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dout + o));
    const float s = warp_sum(fmaf(x.x, y.x, x.y * y.y));
    if (lane == 0) delta[((int64_t)b * H + h) * L + i] = s;
  }
}

template <bool kDrop>
__global__ void __launch_bounds__(128)
attn_bwd_dkdv(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ mask,
              const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ delta,
              __nv_bfloat16* __restrict__ dqkv, int L, int H, const PhiloxArgs drop) {
  __shared__ alignas(16) __nv_bfloat16 sQ[kT * kP], sQt[kT * kP], sO[kT * kP], sOt[kT * kP];
  __shared__ float sL[kT], sD[kT];
  const int k0 = blockIdx.x * kT, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t ldq = (int64_t)3 * H * 64, ldo = (int64_t)H * 64;
  const __nv_bfloat16* base = qkv + (int64_t)b * L * ldq;
  const int64_t sh = ((int64_t)b * H + h) * L;
  // this warp's 16 keys of K and V as A fragments (staged through the Q / dO tiles)
  load_tile(base + (H + h) * 64, ldq, k0, L, sQ, nullptr);
  load_tile(base + (2 * H + h) * 64, ldq, k0, L, sO, nullptr);
  __syncthreads();
  uint32_t kf[4][4], vf[4][4];
  load_afrag(sQ, warp * 16, g, t, kf);
  load_afrag(sO, warp * 16, g, t, vf);
  const int key0 = k0 + warp * 16 + g;
  bool kv[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int key = key0 + 8 * e;
    kv[e] = key < L && (mask == nullptr || mask[(int64_t)b * L + key] != 0);
  }
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[j][e] = dv[j][e] = 0.f;
  [[maybe_unused]] PhiloxKey pk;
  if constexpr (kDrop) pk = philox_key(drop);

  for (int q0 = 0; q0 < L; q0 += kT) {
    __syncthreads();                                        // the previous tiles (or the K / V staging) are consumed
    load_tile(base + h * 64, ldq, q0, L, sQ, sQt);
    load_tile(dout + (int64_t)b * L * ldo + h * 64, ldo, q0, L, sO, sOt);
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
        const uint64_t n = ((uint64_t)sh + (q0 + qc)) * (uint64_t)L + (key0 + 8 * ((i >> 1) & 1));
        km |= dropout_keep(pk, n) ? 1u << i : 0u;
      }
    }
    // S^T (keys x queries) and dP^T = V dO^T
    float p[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) p[j][e] = dp[j][e] = 0.f;
    mma_rows(p, kf, sQ, g, t);
    mma_rows(dp, vf, sO, g, t);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = j * 8 + 2 * t + (e & 1);
        const float pe = kv[e >> 1] ? exp2f(p[j][e] * kScaleLog2 - sL[qc]) : 0.f;
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
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat16* ro = sOt + (j * 8 + g) * kP + k * 16 + 2 * t;
        const __nv_bfloat16* rq = sQt + (j * 8 + g) * kP + k * 16 + 2 * t;
        mma16816(dv[j], pa[k], lds(ro), lds(ro + 8));
        mma16816(dk[j], sa[k], lds(rq), lds(rq + 8));
      }
  }
  __nv_bfloat16* drow = dqkv + (int64_t)b * L * ldq;
  store_rows(dk, drow + (H + h) * 64, ldq, key0, L, t, 0.125f);
  store_rows(dv, drow + (2 * H + h) * 64, ldq, key0, L, t, 1.f);
}

template <bool kDrop>
__global__ void __launch_bounds__(128)
attn_bwd_dq(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ mask,
            const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ delta,
            __nv_bfloat16* __restrict__ dqkv, int L, int H, const PhiloxArgs drop) {
  __shared__ alignas(16) __nv_bfloat16 sK[kT * kP], sKt[kT * kP], sV[kT * kP];
  __shared__ uint8_t sM[kT];
  const int q0 = blockIdx.x * kT, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t ldq = (int64_t)3 * H * 64, ldo = (int64_t)H * 64;
  const __nv_bfloat16* base = qkv + (int64_t)b * L * ldq;
  const int64_t sh = ((int64_t)b * H + h) * L;
  // this warp's 16 queries of Q and dO as A fragments (staged through the K / V tiles)
  load_tile(base + h * 64, ldq, q0, L, sK, nullptr);
  load_tile(dout + (int64_t)b * L * ldo + h * 64, ldo, q0, L, sV, nullptr);
  __syncthreads();
  uint32_t qf[4][4], of[4][4];
  load_afrag(sK, warp * 16, g, t, qf);
  load_afrag(sV, warp * 16, g, t, of);
  const int qr = q0 + warp * 16 + g;
  float rl[2], rd[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int q = qr + 8 * e;
    rl[e] = q < L ? lse[sh + q] : INFINITY;
    rd[e] = q < L ? delta[sh + q] : 0.f;
  }
  float dq[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dq[j][e] = 0.f;
  [[maybe_unused]] PhiloxKey pk;
  if constexpr (kDrop) pk = philox_key(drop);

  for (int kb = 0; kb < L; kb += kT) {
    __syncthreads();
    load_tile(base + (H + h) * 64, ldq, kb, L, sK, sKt);
    load_tile(base + (2 * H + h) * 64, ldq, kb, L, sV, nullptr);
    if (threadIdx.x < kT) {
      const int key = kb + threadIdx.x;
      sM[threadIdx.x] = (key < L && (mask == nullptr || mask[(int64_t)b * L + key] != 0)) ? 1 : 0;
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = dp[j][e] = 0.f;
    mma_rows(s, qf, sK, g, t);
    mma_rows(dp, of, sV, g, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      [[maybe_unused]] uint32_t keep[2];
      if constexpr (kDrop) {
#pragma unroll
        for (int r = 0; r < 2; ++r)
          keep[r] = dropout_keep2(pk, ((uint64_t)sh + (qr + 8 * r)) * (uint64_t)L + (kb + j * 8 + 2 * t));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = j * 8 + 2 * t + (e & 1);
        const float pe = sM[kc] ? exp2f(s[j][e] * kScaleLog2 - rl[e >> 1]) : 0.f;
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
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat16* rk = sKt + (j * 8 + g) * kP + k * 16 + 2 * t;
        mma16816(dq[j], sa[k], lds(rk), lds(rk + 8));
      }
  }
  store_rows(dq, dqkv + (int64_t)b * L * ldq + h * 64, ldq, qr, L, t, 0.125f);
}

}  // namespace

const char* attention_bwd(const void* qkv, const uint8_t* mask, const void* out, const float* lse, const void* dout,
                          void* dqkv, float* delta, int B, int L, int H, cudaStream_t stream, const PhiloxArgs* drop) {
  if (!attention_supported(B, L, H, 64)) return "attention_bwd: unsupported shape (head dim 64, 1 <= L <= 512)";
  const auto* q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  const auto* o = reinterpret_cast<const __nv_bfloat16*>(out);
  const auto* d = reinterpret_cast<const __nv_bfloat16*>(dout);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  const int64_t rows = (int64_t)B * L;
  attn_bwd_delta<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(o, d, delta, B, L, H);
  const dim3 grid((L + kT - 1) / kT, H, B);
  if (drop != nullptr) {
    attn_bwd_dkdv<true><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, *drop);
    attn_bwd_dq<true><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, *drop);
  } else {
    attn_bwd_dkdv<false><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, PhiloxArgs{});
    attn_bwd_dq<false><<<grid, 128, 0, stream>>>(q, mask, d, lse, delta, dq, L, H, PhiloxArgs{});
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace edl
