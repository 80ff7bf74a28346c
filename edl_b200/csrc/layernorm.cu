// LayerNorm over the hidden dimension, and the embedding sum + LayerNorm of a BERT / ERNIE encoder's input (inference).
// One warp per row: a lane holds up to four 16-byte chunks (8 bf16) of the row in registers, so the row is read once
// and the variance is the two-pass sum of (x - mean)^2 over the registers.  C % 8 == 0, C <= 1024.
//
// The quantising variants (template argument Q) also write e4m3 bytes q [rows, C] and fp32 scales sa [ceil(C/128), rows]
// of the stored bf16 y, for the block-scaled FP8 GEMM that reads it: a 128-element block is one half-warp's chunk c, so
// its max|y| is the half-warp shuffle of quantize_e4m3_blocks (gemm_fp8.cu) and the bytes and scales are those it writes.
//
// Backward (training): one warp per row over a fixed grid of layernorm_bwd_ctas(rows) CTAs (a function of the row count
// only).  The row statistics are recomputed from the saved pre-LN input exactly as the forward forms them, then
// dx = rstd (g - mean(g) - xhat mean(g xhat)) with g = dy gamma.  Each lane keeps dgamma / dbeta of its columns in
// registers over the rows of its warp; a CTA sums its eight warps in warp order into one fp32 partial row, and a second
// kernel adds the partials of all CTAs in CTA order: no atomics, bitwise reproducible.  The embedding variant (EMB)
// re-gathers word + pos + seg the way the forward does and writes the row gradient dE in fp32.
// Dropout on the embedding-LayerNorm output (training, DROP): the forward multiplies y by Z = keep * 1 / (1 - p) of the
// mask of philox.cuh at flat index row * C + col before the bf16 store, and the backward applies the same Z to dy as
// it loads it.  Plain LayerNorm has no dropout.
// Budgets (ptxas -v, 256 threads): layernorm_bwd_kernel 159 registers, embedding variant 161, no spills; 32 KB static
// shared memory for the partial sums.
#include <cuda_fp8.h>

#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace edl {
namespace {

constexpr int kLnWarps = 8;
constexpr int kLnChunks = kLnMaxC / 256;     // 16-byte chunks per lane

// Q: where the quantised copy goes (q: this row's C bytes; sa: the row's first scale, one scale every `rows` floats)
struct LnQuant {
  uint8_t* q;
  float* sa;
  int64_t rows;
};

// y[e] *= Z of the eight elements at flat mask index n .. n + 7 (n % 8 == 0)
EDL_DEVICE void dropout8(const PhiloxKey& k, uint64_t n, float (&y)[8]) {
  const uint4 w0 = philox_group(k, n >> 2), w1 = philox_group(k, (n >> 2) + 1);
  const uint32_t w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
  for (int e = 0; e < 8; ++e) y[e] = w[e] >= k.threshold ? y[e] * k.scale : 0.f;
}

// x: this lane's chunks of the row (chunk c of the lane is columns (c * 32 + lane) * 8 ..), n8 = C / 8.  DROP: dropout
// on the stored y with the mask indices nrow + col.
template <bool Q = false, bool DROP = false>
EDL_DEVICE void ln_store(float (&x)[kLnChunks][8], int lane, int n8, int C, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ yrow,
                         [[maybe_unused]] const LnQuant& qo = LnQuant{}, [[maybe_unused]] const PhiloxKey& pk = {},
                         [[maybe_unused]] uint64_t nrow = 0) {
  static_assert(!(Q && DROP), "dropout: bf16 output only");
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c)
    if (c * 32 + lane < n8)
#pragma unroll
      for (int e = 0; e < 8; ++e) s += x[c][e];
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c)
    if (c * 32 + lane < n8)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = x[c][e] - mean;
        q = fmaf(d, d, q);
      }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
  if constexpr (Q) {
    // every lane of a live chunk takes part in the shuffles; lanes past C hold zeros (a short tail block)
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      if (c * 32 >= n8) break;
      const int k = c * 32 + lane;
      const bool live = k < n8;
      float y[8];
      if (live) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * k), b1 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * k + 1);
        const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = fmaf((x[c][e] - mean) * rstd, g[e], bb[e]);
        const bf16x8 pk = pack8(y);
        st_vec(yrow + k * 8, pk);
        unpack8(pk, y);                                      // quantise the stored bf16 values
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = 0.f;
      }
      float amax = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(y[e]));
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      const float s = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
      const int b = k >> 4;                                   // = 2 c + lane / 16
      if ((lane & 15) == 0 && b * 16 < n8) qo.sa[(int64_t)b * qo.rows] = s;
      if (live) {
        uint8_t o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (uint8_t)__nv_cvt_float_to_fp8(__fdiv_rn(y[e], s), __NV_SATFINITE, __NV_E4M3);
        *reinterpret_cast<uint2*>(qo.q + k * 8) = *reinterpret_cast<const uint2*>(o);
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k >= n8) continue;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * k), b1 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * k + 1);
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = fmaf((x[c][e] - mean) * rstd, g[e], bb[e]);
      if constexpr (DROP) dropout8(pk, nrow + k * 8, y);
      st_vec(yrow + k * 8, pack8(y));
    }
  }
}

template <bool Q>
__global__ void __launch_bounds__(kLnWarps * 32)
layernorm_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps, uint8_t* __restrict__ q, float* __restrict__ sa) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int n8 = C / 8;
  float v[kLnChunks][8];
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c) {
    const int k = c * 32 + lane;
    if (k < n8) {
      float f[8];
      unpack8(ld_vec(x + r * C + k * 8), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[c][e] = f[e];
    }
  }
  ln_store<Q>(v, lane, n8, C, gamma, beta, eps, y + r * C, LnQuant{q + r * C, sa + r, rows});
}

template <bool Q, bool DROP = false>
__global__ void __launch_bounds__(kLnWarps * 32)
embedding_layernorm_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos_ids,
                           const int64_t* __restrict__ seg_ids, const __nv_bfloat16* __restrict__ word, int64_t n_word,
                           const __nv_bfloat16* __restrict__ pos, int64_t n_pos, const __nv_bfloat16* __restrict__ seg,
                           int64_t n_seg, const float* __restrict__ gamma, const float* __restrict__ beta,
                           __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps, int* err,
                           uint8_t* __restrict__ q, float* __restrict__ sa, const PhiloxArgs drop) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int n8 = C / 8;
  const int64_t iw = ids[r], ip = pos_ids[r], is = seg_ids[r];
  const bool okw = iw >= 0 && iw < n_word, okp = ip >= 0 && ip < n_pos, oks = is >= 0 && is < n_seg;
  if (!(okw && okp && oks) && lane == 0) atomicExch(err, 1);
  float v[kLnChunks][8];
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c) {
    const int k = c * 32 + lane;
    if (k < n8) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[c][e] = 0.f;
      float f[8];
      if (okw) {
        unpack8(ld_vec(word + iw * C + k * 8), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[c][e] += f[e];
      }
      if (okp) {
        unpack8(ld_vec(pos + ip * C + k * 8), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[c][e] += f[e];
      }
      if (oks) {
        unpack8(ld_vec(seg + is * C + k * 8), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[c][e] += f[e];
      }
    }
  }
  if constexpr (DROP)
    ln_store<Q, true>(v, lane, n8, C, gamma, beta, eps, y + r * C, LnQuant{}, philox_key(drop), (uint64_t)r * C);
  else
    ln_store<Q>(v, lane, n8, C, gamma, beta, eps, y + r * C, LnQuant{q + r * C, sa + r, rows});
}

constexpr int kLnBwdMaxCtas = 264;

// v[c][e] = this lane's columns of the pre-LN row: the bf16 input, or the forward's embedding sum
template <bool EMB>
EDL_DEVICE void ln_bwd_row(const __nv_bfloat16* __restrict__ x, const int64_t* __restrict__ ids,
                           const int64_t* __restrict__ pos_ids, const int64_t* __restrict__ seg_ids,
                           const __nv_bfloat16* __restrict__ word, int64_t n_word, const __nv_bfloat16* __restrict__ pos,
                           int64_t n_pos, const __nv_bfloat16* __restrict__ seg, int64_t n_seg, int64_t r, int lane,
                           int n8, int C, float (&v)[kLnChunks][8]) {
  if constexpr (EMB) {
    const int64_t iw = ids[r], ip = pos_ids[r], is = seg_ids[r];
    const bool okw = iw >= 0 && iw < n_word, okp = ip >= 0 && ip < n_pos, oks = is >= 0 && is < n_seg;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k < n8) {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[c][e] = 0.f;
        float f[8];
        if (okw) {
          unpack8(ld_vec(word + iw * C + k * 8), f);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[c][e] += f[e];
        }
        if (okp) {
          unpack8(ld_vec(pos + ip * C + k * 8), f);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[c][e] += f[e];
        }
        if (oks) {
          unpack8(ld_vec(seg + is * C + k * 8), f);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[c][e] += f[e];
        }
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k < n8) unpack8(ld_vec(x + r * C + k * 8), v[c]);
    }
  }
}

template <bool EMB, bool DROP = false>
__global__ void __launch_bounds__(kLnWarps * 32)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, const int64_t* __restrict__ ids,
                     const int64_t* __restrict__ pos_ids, const int64_t* __restrict__ seg_ids,
                     const __nv_bfloat16* __restrict__ word, int64_t n_word, const __nv_bfloat16* __restrict__ pos,
                     int64_t n_pos, const __nv_bfloat16* __restrict__ seg, int64_t n_seg,
                     const __nv_bfloat16* __restrict__ dy, const float* __restrict__ gamma, void* __restrict__ dx,
                     float* __restrict__ part, int64_t rows, int C, float eps, const PhiloxArgs drop) {
  static_assert(EMB || !DROP, "dropout: embedding-LayerNorm only");
  __shared__ float red[kLnWarps][kLnMaxC];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n8 = C / 8;
  float dg[kLnChunks][8], db[kLnChunks][8];
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c)
#pragma unroll
    for (int e = 0; e < 8; ++e) dg[c][e] = db[c][e] = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * kLnWarps + w; r < rows; r += (int64_t)gridDim.x * kLnWarps) {
    float v[kLnChunks][8], d[kLnChunks][8];
    ln_bwd_row<EMB>(x, ids, pos_ids, seg_ids, word, n_word, pos, n_pos, seg, n_seg, r, lane, n8, C, v);
    // the forward's statistics, formed the same way
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c)
      if (c * 32 + lane < n8)
#pragma unroll
        for (int e = 0; e < 8; ++e) s += v[c][e];
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c)
      if (c * 32 + lane < n8)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float t = v[c][e] - mean;
          q = fmaf(t, t, q);
        }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k >= n8) continue;
      unpack8(ld_vec(dy + r * C + k * 8), d[c]);
      if constexpr (DROP) dropout8(philox_key(drop), (uint64_t)r * C + k * 8, d[c]);
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * k + 1);
      const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        v[c][e] = (v[c][e] - mean) * rstd;                  // xhat
        dg[c][e] = fmaf(d[c][e], v[c][e], dg[c][e]);
        db[c][e] += d[c][e];
        d[c][e] *= gm[e];                                    // g = dy gamma
        sg += d[c][e];
        sgx = fmaf(d[c][e], v[c][e], sgx);
      }
    }
    const float mg = warp_sum(sg) / (float)C, mgx = warp_sum(sgx) / (float)C;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k >= n8) continue;
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * (d[c][e] - mg - v[c][e] * mgx);
      if constexpr (EMB) {
        float4* p = reinterpret_cast<float4*>(static_cast<float*>(dx) + r * C + k * 8);
        p[0] = make_float4(o[0], o[1], o[2], o[3]);
        p[1] = make_float4(o[4], o[5], o[6], o[7]);
      } else {
        st_vec(static_cast<__nv_bfloat16*>(dx) + r * C + k * 8, pack8(o));
      }
    }
  }
  // the CTA's partial: its warps summed in warp order, dgamma then dbeta
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int k = c * 32 + lane;
      if (k < n8)
#pragma unroll
        for (int e = 0; e < 8; ++e) red[w][k * 8 + e] = pass == 0 ? dg[c][e] : db[c][e];
    }
    __syncthreads();
    for (int col = threadIdx.x; col < C; col += kLnWarps * 32) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < kLnWarps; ++i) t += red[i][col];
      part[((int64_t)blockIdx.x * 2 + pass) * C + col] = t;
    }
    __syncthreads();
  }
}

// dgamma / dbeta: the partials of all CTAs in CTA order
__global__ void __launch_bounds__(256)
layernorm_bwd_reduce(const float* __restrict__ part, int ctas, int C, float* __restrict__ dgamma,
                     float* __restrict__ dbeta) {
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col >= 2 * C) return;
  const int pass = col / C, c = col % C;
  float t = 0.f;
  for (int i = 0; i < ctas; ++i) t += part[((int64_t)i * 2 + pass) * C + c];
  (pass == 0 ? dgamma : dbeta)[c] = t;
}

}  // namespace

int layernorm_bwd_ctas(int64_t rows) {
  const int64_t n = (rows + kLnWarps - 1) / kLnWarps;
  return (int)(n < 1 ? 1 : (n < kLnBwdMaxCtas ? n : kLnBwdMaxCtas));
}

void layernorm_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* part, float* dgamma,
                   float* dbeta, int64_t rows, int C, float eps, cudaStream_t s) {
  const int ctas = layernorm_bwd_ctas(rows);
  layernorm_bwd_kernel<false><<<ctas, kLnWarps * 32, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0, nullptr, 0,
      reinterpret_cast<const __nv_bfloat16*>(dy), gamma, dx, part, rows, C, eps, PhiloxArgs{});
  layernorm_bwd_reduce<<<(2 * C + 255) / 256, 256, 0, s>>>(part, ctas, C, dgamma, dbeta);
}

void embedding_layernorm_bwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                             int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                             const void* dy, const float* gamma, float* dE, float* part, float* dgamma, float* dbeta,
                             int64_t rows, int C, float eps, cudaStream_t s, const PhiloxArgs* drop) {
  const int ctas = layernorm_bwd_ctas(rows);
  auto kern = drop != nullptr ? layernorm_bwd_kernel<true, true> : layernorm_bwd_kernel<true>;
  kern<<<ctas, kLnWarps * 32, 0, s>>>(
      nullptr, ids, pos_ids, seg_ids, reinterpret_cast<const __nv_bfloat16*>(word), n_word,
      reinterpret_cast<const __nv_bfloat16*>(pos), n_pos, reinterpret_cast<const __nv_bfloat16*>(seg), n_seg,
      reinterpret_cast<const __nv_bfloat16*>(dy), gamma, dE, part, rows, C, eps, drop != nullptr ? *drop : PhiloxArgs{});
  layernorm_bwd_reduce<<<(2 * C + 255) / 256, 256, 0, s>>>(part, ctas, C, dgamma, dbeta);
}

bool layernorm_supported(int C) { return C >= 8 && C <= kLnMaxC && C % 8 == 0; }

void layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps,
                   cudaStream_t s) {
  if (rows <= 0) return;
  layernorm_kernel<false><<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps, nullptr,
      nullptr);
}

void layernorm_e4m3_fwd(const void* x, const float* gamma, const float* beta, void* y, void* q, float* sa, int64_t rows,
                        int C, float eps, cudaStream_t s) {
  if (rows <= 0) return;
  layernorm_kernel<true><<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps,
      reinterpret_cast<uint8_t*>(q), sa);
}

void embedding_layernorm_fwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                             int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                             const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps, int* err,
                             cudaStream_t s, const PhiloxArgs* drop) {
  if (rows <= 0) return;
  auto kern = drop != nullptr ? embedding_layernorm_kernel<false, true> : embedding_layernorm_kernel<false>;
  kern<<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      ids, pos_ids, seg_ids, reinterpret_cast<const __nv_bfloat16*>(word), n_word,
      reinterpret_cast<const __nv_bfloat16*>(pos), n_pos, reinterpret_cast<const __nv_bfloat16*>(seg), n_seg, gamma,
      beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps, err, nullptr, nullptr,
      drop != nullptr ? *drop : PhiloxArgs{});
}

void embedding_layernorm_e4m3_fwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                                  int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                                  const float* gamma, const float* beta, void* y, void* q, float* sa, int64_t rows, int C,
                                  float eps, int* err, cudaStream_t s) {
  if (rows <= 0) return;
  embedding_layernorm_kernel<true><<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      ids, pos_ids, seg_ids, reinterpret_cast<const __nv_bfloat16*>(word), n_word,
      reinterpret_cast<const __nv_bfloat16*>(pos), n_pos, reinterpret_cast<const __nv_bfloat16*>(seg), n_seg, gamma,
      beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps, err, reinterpret_cast<uint8_t*>(q), sa, PhiloxArgs{});
}

}  // namespace edl
