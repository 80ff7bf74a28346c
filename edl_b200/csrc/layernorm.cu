// LayerNorm over the hidden dimension, and the embedding sum + LayerNorm of a BERT / ERNIE encoder's input (inference).
// One warp per row: a lane holds up to four 16-byte chunks (8 bf16) of the row in registers, so the row is read once
// and the variance is the two-pass sum of (x - mean)^2 over the registers.  C % 8 == 0, C <= 1024.
#include "common.cuh"
#include "kernels.h"

namespace edl {
namespace {

constexpr int kLnWarps = 8;
constexpr int kLnChunks = kLnMaxC / 256;     // 16-byte chunks per lane

// x: this lane's chunks of the row (chunk c of the lane is columns (c * 32 + lane) * 8 ..), n8 = C / 8
EDL_DEVICE void ln_store(float (&x)[kLnChunks][8], int lane, int n8, int C, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ yrow) {
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
    st_vec(yrow + k * 8, pack8(y));
  }
}

__global__ void __launch_bounds__(kLnWarps * 32)
layernorm_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps) {
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
  ln_store(v, lane, n8, C, gamma, beta, eps, y + r * C);
}

__global__ void __launch_bounds__(kLnWarps * 32)
embedding_layernorm_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos_ids,
                           const int64_t* __restrict__ seg_ids, const __nv_bfloat16* __restrict__ word, int64_t n_word,
                           const __nv_bfloat16* __restrict__ pos, int64_t n_pos, const __nv_bfloat16* __restrict__ seg,
                           int64_t n_seg, const float* __restrict__ gamma, const float* __restrict__ beta,
                           __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps, int* err) {
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
  ln_store(v, lane, n8, C, gamma, beta, eps, y + r * C);
}

}  // namespace

bool layernorm_supported(int C) { return C >= 8 && C <= kLnMaxC && C % 8 == 0; }

void layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps,
                   cudaStream_t s) {
  if (rows <= 0) return;
  layernorm_kernel<<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps);
}

void embedding_layernorm_fwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                             int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                             const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps, int* err,
                             cudaStream_t s) {
  if (rows <= 0) return;
  embedding_layernorm_kernel<<<(unsigned)((rows + kLnWarps - 1) / kLnWarps), kLnWarps * 32, 0, s>>>(
      ids, pos_ids, seg_ids, reinterpret_cast<const __nv_bfloat16*>(word), n_word,
      reinterpret_cast<const __nv_bfloat16*>(pos), n_pos, reinterpret_cast<const __nv_bfloat16*>(seg), n_seg, gamma,
      beta, reinterpret_cast<__nv_bfloat16*>(y), rows, C, eps, err);
}

}  // namespace edl
