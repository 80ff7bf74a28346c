// Shared device helpers for the edl_b200 sm_90a kernels.
// Pure CUDA (no torch headers) so each .cu compiles in seconds with nvcc.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define EDL_DEVICE __device__ __forceinline__

namespace edl {

constexpr int kNumSMs = 132;  // H100 SXM

struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};

EDL_DEVICE void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

EDL_DEVICE bf16x8 pack8(const float (&f)[8]) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

// 128-bit streaming load (read-only path, no L1 allocation) for one-touch data.  NOT volatile: the
// compiler may hoist / batch it freely (the data is never written by the same kernel).
EDL_DEVICE bf16x8 ld_stream(const void* ptr) {
  int4 r;
  asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
      : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
      : "l"(ptr));
  return *reinterpret_cast<bf16x8*>(&r);
}

// Four independent 128-bit streaming loads issued back to back from ONE asm block: guarantees the
// memory-level parallelism (ptxas otherwise interleaves each load with the math that consumes it,
// which measured at 10% of HBM bandwidth on the BN kernels -- profiles/ round-1 ncu capture).
EDL_DEVICE void ld_stream_x4(const void* p0, const void* p1, const void* p2, const void* p3,
                             bf16x8 (&v)[4]) {
  int4 a, b, c, d;
  asm volatile(
      "ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%16];\n\t"
      "ld.global.nc.L1::no_allocate.v4.s32 {%4,%5,%6,%7}, [%17];\n\t"
      "ld.global.nc.L1::no_allocate.v4.s32 {%8,%9,%10,%11}, [%18];\n\t"
      "ld.global.nc.L1::no_allocate.v4.s32 {%12,%13,%14,%15}, [%19];"
      : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w),
        "=r"(c.x), "=r"(c.y), "=r"(c.z), "=r"(c.w), "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w)
      : "l"(p0), "l"(p1), "l"(p2), "l"(p3));
  v[0] = *reinterpret_cast<bf16x8*>(&a);
  v[1] = *reinterpret_cast<bf16x8*>(&b);
  v[2] = *reinterpret_cast<bf16x8*>(&c);
  v[3] = *reinterpret_cast<bf16x8*>(&d);
}
EDL_DEVICE bf16x8 ld_vec(const void* ptr) { return *reinterpret_cast<const bf16x8*>(ptr); }
EDL_DEVICE void st_vec(void* ptr, const bf16x8& v) { *reinterpret_cast<bf16x8*>(ptr) = v; }
EDL_DEVICE void st_stream(void* ptr, const bf16x8& v) {
  const int4& r = *reinterpret_cast<const int4*>(&v);
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(ptr), "r"(r.x),
               "r"(r.y), "r"(r.z), "r"(r.w));
}

EDL_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// fp32 reductions into global memory.  Hot accumulators (per-channel BatchNorm sums: a few KB hit by
// every CTA) are limited by the number of reduction REQUESTS the L2 can retire when all SMs hammer the
// same ~1k addresses, so four floats go in one request.
EDL_DEVICE void red_add_v4(float* dst, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// dst[0..7] += v[0..7]; vectorised when dst is 16-byte aligned
EDL_DEVICE void red_add8(float* dst, const float* v) {
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    red_add_v4(dst, v[0], v[1], v[2], v[3]);
    red_add_v4(dst + 4, v[4], v[5], v[6], v[7]);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) atomicAdd(dst + i, v[i]);
  }
}

// dst[0..3] = bf16(v), or bf16(dst + v) when accumulating (the sum in fp32, one rounding); dst 8-byte aligned
EDL_DEVICE void store_bf16x4(__nv_bfloat16* dst, float4 v, bool accumulate) {
  if (accumulate) {
    const uint2 old = *reinterpret_cast<const uint2*>(dst);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&old.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&old.y));
    v.x += a.x; v.y += a.y; v.z += b.x; v.w += b.y;
  }
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
  const __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 packed;
  packed.x = *reinterpret_cast<const uint32_t*>(&lo);
  packed.y = *reinterpret_cast<const uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(dst) = packed;
}

// The first min(n, 4) elements of v into dst (+= when accumulating) with 2-byte stores: the last columns of a row, or
// rows that are not 8-byte aligned.
EDL_DEVICE void store_bf16_tail(__nv_bfloat16* dst, float4 v, int n, bool accumulate) {
  const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i >= n) break;
    dst[i] = __float2bfloat16_rn(accumulate ? e[i] + __bfloat162float(dst[i]) : e[i]);
  }
}

EDL_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Programmatic dependent launch (PDL).  A kernel launched with the programmatic-stream-serialization
// attribute (launch.h) may start while its predecessor in the stream is still running: everything up to
// pdl_wait() -- barrier init, tensor-map prefetch -- overlaps the predecessor's tail, and
// pdl_wait() returns once the predecessor grid has completed and its memory is visible.  Both instructions are
// no-ops for a normally launched kernel.  RULE: a kernel launched through launch_pdl() must execute pdl_wait()
// before its first access to global memory.
EDL_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
EDL_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename T>
EDL_DEVICE T ceil_div(T a, T b) {
  return (a + b - 1) / b;
}

}  // namespace edl
