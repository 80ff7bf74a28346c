// y = Z o x for bf16 tensors of any length (Z = keep * scale, the mask of philox.cuh over the flat index): the public
// ops.dropout and the residual-branch backward of the Transformer student (dh_branch = Z o dh).  A thread takes eight
// consecutive elements, two Philox groups; with both pointers 16-byte aligned the body moves them as one 16-byte vector,
// and the tail (or an unaligned tensor) goes element by element.
#include "philox.cuh"

namespace edl {
namespace {

__global__ void __launch_bounds__(256)
dropout_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n, bool vec,
               const PhiloxArgs drop) {
  const int64_t i0 = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 8;
  if (i0 >= n) return;
  const PhiloxKey k = philox_key(drop);
  const uint4 w0 = philox_group(k, (uint64_t)i0 >> 2), w1 = philox_group(k, ((uint64_t)i0 >> 2) + 1);
  const uint32_t w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
  if (vec && i0 + 8 <= n) {
    float f[8];
    unpack8(ld_vec(x + i0), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = w[e] >= k.threshold ? f[e] * k.scale : 0.f;
    st_vec(y + i0, pack8(f));
    return;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e)
    if (i0 + e < n) y[i0 + e] = __float2bfloat16_rn(w[e] >= k.threshold ? __bfloat162float(x[i0 + e]) * k.scale : 0.f);
}

}  // namespace

void dropout_apply(const void* x, void* y, int64_t n, const PhiloxArgs& drop, cudaStream_t s) {
  if (n <= 0) return;
  const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  const int64_t threads = (n + 7) / 8;
  dropout_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                                    reinterpret_cast<__nv_bfloat16*>(y), n, vec, drop);
}

}  // namespace edl
