// Bulk-async (TMA 1-D, cp.async.bulk) streaming versions of the NHWC batch-norm kernels.
//
// Why: the register-based BN kernels (bn.cu) reached only 10-17 % of HBM bandwidth in the round-1
// ncu capture: ptxas interleaves every 128-bit load with the math consuming it, so a warp
// never has more than 2 loads in flight and register pressure caps occupancy at 16 warps/SM.
// Here one producer lane per CTA streams 16 KB chunks of each operand into a 4-stage shared-memory
// ring with cp.async.bulk + mbarrier transaction counts (up to 192 KB in flight per SM, zero
// registers), and 16 consumer warps read the staged chunk with conflict-free 128-bit LDS.
// One persistent CTA per SM; chunks are dealt round-robin.
//
// Requirements: C a power of two in [8, 4096] (so every thread keeps a fixed 8-channel group and
// can hold the per-channel coefficients / accumulators in registers).  Other shapes use bn.cu.
#include "common.cuh"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kConsumers = 512;                 // 16 consumer warps
constexpr int kThreads = kConsumers + 32;       // + 1 producer warp
constexpr int kChunkElems = 8192;               // bf16 elements per operand per stage (16 KB)
constexpr int kChunkBytes = kChunkElems * 2;
constexpr int kStages = 4;
constexpr int kVecPerThread = kChunkElems / 8 / kConsumers;  // 2

EDL_DEVICE void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          ptx::smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(ptx::smem_u32(bar))
      : "memory");
}

template <int NT>
struct Ring {
  uint8_t* data;        // [kStages][NT][kChunkBytes]
  uint64_t* full;       // [kStages]
  uint64_t* empty;      // [kStages]
  EDL_DEVICE uint8_t* buf(int stage, int t) const { return data + ((size_t)stage * NT + t) * kChunkBytes; }
};

template <int NT>
EDL_DEVICE Ring<NT> ring_init(uint8_t* smem_raw) {
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  Ring<NT> r;
  r.data = smem;
  r.full = reinterpret_cast<uint64_t*>(smem + (size_t)kStages * NT * kChunkBytes);
  r.empty = r.full + kStages;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&r.full[s], 1);
      ptx::mbar_init(&r.empty[s], kConsumers / 32);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch: the ring set-up above overlapped the previous kernel's tail; every kernel of
  // this file calls ring_init() before its first global access
  pdl_wait();
  pdl_launch_dependents();
  return r;
}

template <int NT>
constexpr size_t ring_smem_bytes() {
  return (size_t)kStages * NT * kChunkBytes + 2 * kStages * sizeof(uint64_t) + 128;
}

// Producer loop (one lane of the producer warp).  Operand MASK_T (if >= 0) is a ReLU mask with one bit per element
// (uint8 [M, C / 8]): 1/16 of a bf16 operand's bytes, which stay a multiple of 16 when C % 128 == 0.
template <int NT, int MASK_T = -1>
EDL_DEVICE void produce(const Ring<NT>& r, const void* const (&src)[NT], int64_t total_elems, int64_t n_chunks) {
  int it = 0;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x, ++it) {
    const int s = it % kStages;
    const uint32_t ph = (it / kStages) & 1;
    ptx::mbar_wait(&r.empty[s], ph ^ 1);
    const int64_t off = ch * kChunkElems;
    int64_t rem = total_elems - off;
    const uint32_t bytes = (uint32_t)((rem < kChunkElems ? rem : kChunkElems) * 2);
    ptx::mbar_arrive_expect_tx(&r.full[s], MASK_T < 0 ? bytes * NT : bytes * (NT - 1) + bytes / 16);
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      if (t == MASK_T)
        bulk_load(r.buf(s, t), reinterpret_cast<const uint8_t*>(src[t]) + off / 8, bytes / 16, &r.full[s]);
      else
        bulk_load(r.buf(s, t), reinterpret_cast<const __nv_bfloat16*>(src[t]) + off, bytes, &r.full[s]);
    }
  }
}

// Consumer loop: body(global_elem_offset, smem pointers of the NT operands); the pointer of a mask operand points at
// the vector's mask byte
template <int NT, int MASK_T = -1, class Body>
EDL_DEVICE void consume(const Ring<NT>& r, int64_t total_elems, int64_t n_chunks, Body body) {
  const int tid = threadIdx.x;
  int it = 0;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x, ++it) {
    const int s = it % kStages;
    const uint32_t ph = (it / kStages) & 1;
    ptx::mbar_wait(&r.full[s], ph);
    const int64_t off = ch * kChunkElems;
    int64_t rem = total_elems - off;
    const int valid_vecs = (int)((rem < kChunkElems ? rem : kChunkElems) / 8);
#pragma unroll
    for (int k = 0; k < kVecPerThread; ++k) {
      const int v = tid + k * kConsumers;
      if (v < valid_vecs) {
        const bf16x8* ptrs[NT];
#pragma unroll
        for (int t = 0; t < NT; ++t)
          ptrs[t] = t == MASK_T ? reinterpret_cast<const bf16x8*>(r.buf(s, t) + v)
                                : reinterpret_cast<const bf16x8*>(r.buf(s, t)) + v;
        body(off + (int64_t)v * 8, ptrs);
      }
    }
    __syncwarp();
    if ((tid & 31) == 0) ptx::mbar_arrive(&r.empty[s]);
  }
}

// Sum `acc[NV]` over all consumer threads that share a channel group (tid % cvecs); result valid in
// threads tid < cvecs.  `scratch` must hold kConsumers * NV floats and the pipeline must be drained.
template <int NV>
EDL_DEVICE void reduce_groups(float (&acc)[NV], int cvecs, float* scratch, bool is_consumer) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (is_consumer) {
#pragma unroll
    for (int k = 0; k < NV; ++k) scratch[k * kConsumers + tid] = acc[k];
  }
  __syncthreads();
  for (int stride = kConsumers >> 1; stride >= cvecs; stride >>= 1) {
    if (is_consumer && tid < stride) {
#pragma unroll
      for (int k = 0; k < NV; ++k) scratch[k * kConsumers + tid] += scratch[k * kConsumers + tid + stride];
    }
    __syncthreads();
  }
  if (is_consumer && tid < cvecs) {
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = scratch[k * kConsumers + tid];
  }
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
bn_stats_stream_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ sums, int64_t total, int C) {
  extern __shared__ uint8_t smem_raw[];
  Ring<1> r = ring_init<1>(smem_raw);
  const int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  const int tid = threadIdx.x;
  const bool consumer = tid < kConsumers;
  const int cvecs = C / 8;
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  if (!consumer) {
    if (tid == kConsumers) {
      const void* src[1] = {x};
      produce<1>(r, src, total, n_chunks);
    }
  } else {
    consume<1>(r, total, n_chunks, [&](int64_t, const bf16x8* const (&p)[1]) {
      float f[8];
      unpack8(*p[0], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i] += f[i];
        acc[8 + i] = fmaf(f[i], f[i], acc[8 + i]);
      }
    });
  }
  reduce_groups<16>(acc, cvecs, reinterpret_cast<float*>(r.data), consumer);
  if (consumer && tid < cvecs) {
    red_add8(&sums[tid * 8], acc);
    red_add8(&sums[C + tid * 8], acc + 8);
  }
}

// mask (optional, HAS_RES only): uint8 [M, C / 8], bit b of byte j = (stored y[:, 8 j + b] > 0), C % 128 == 0
template <bool HAS_RES>
__global__ void __launch_bounds__(kThreads, 1)
bn_apply_stream_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                       __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ mask, const float* __restrict__ sums,
                       const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ running_mean, float* __restrict__ running_var,
                       float* __restrict__ saved_mean, float* __restrict__ saved_rstd, int64_t total, int C,
                       float eps, float momentum, int relu) {
  extern __shared__ uint8_t smem_raw[];
  constexpr int NT = HAS_RES ? 2 : 1;
  Ring<NT> r = ring_init<NT>(smem_raw);
  const int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  const int tid = threadIdx.x;
  const int cvecs = C / 8;
  if (tid >= kConsumers) {
    if (tid == kConsumers) {
      const void* src[NT];
      src[0] = x;
      if (HAS_RES) src[NT - 1] = res;
      produce<NT>(r, src, total, n_chunks);
    }
    return;
  }
  const int c0 = (tid % cvecs) * 8;
  const int64_t M = total / C;
  const float inv_m = 1.f / (float)M;
  float scale[8], shift[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float mean = sums[c0 + i] * inv_m;
    const float var = fmaxf(sums[C + c0 + i] * inv_m - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    scale[i] = gamma[c0 + i] * rstd;
    shift[i] = beta[c0 + i] - mean * scale[i];
    if (blockIdx.x == 0 && tid < cvecs) {
      saved_mean[c0 + i] = mean;
      saved_rstd[c0 + i] = rstd;
      if (running_mean != nullptr) {
        const float unbiased = M > 1 ? var * ((float)M / (float)(M - 1)) : var;
        running_mean[c0 + i] = (1.f - momentum) * running_mean[c0 + i] + momentum * mean;
        running_var[c0 + i] = (1.f - momentum) * running_var[c0 + i] + momentum * unbiased;
      }
    }
  }
  consume<NT>(r, total, n_chunks, [&](int64_t goff, const bf16x8* const (&p)[NT]) {
    float f[8];
    unpack8(*p[0], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = fmaf(f[i], scale[i], shift[i]);
    if (HAS_RES) {
      float g[8];
      unpack8(*p[NT - 1], g);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] += g[i];
    }
    if (relu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = fmaxf(f[i], 0.f);
    }
    const bf16x8 o = pack8(f);
    st_vec(y + goff, o);
    if (HAS_RES && mask != nullptr) {
      // the bits test the STORED bf16 values (an fp32 result that rounds to a bf16 zero is masked).  Consecutive lanes
      // hold consecutive vectors and the valid vectors of a chunk are a multiple of 16 (C >= 128), so every group of
      // four lanes is complete: three shuffles gather four mask bytes into its first lane, which stores them as a word.
      unpack8(o, f);
      uint32_t b = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) b |= (f[i] > 0.f ? 1u : 0u) << i;
      const int lane = tid & 31;
      const unsigned grp = 0xFu << (lane & ~3);
#pragma unroll
      for (int d = 1; d < 4; ++d) b |= __shfl_down_sync(grp, b & 0xFFu, d, 4) << (8 * d);
      if ((lane & 3) == 0) *reinterpret_cast<uint32_t*>(mask + goff / 8) = b;
    }
  });
}

struct Coef {
  float mean[8], rstd[8], scale[8], shift[8];
};

EDL_DEVICE void load_coef(Coef& k, const float* saved_mean, const float* saved_rstd, const float* gamma,
                          const float* beta, int c0) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    k.mean[i] = saved_mean[c0 + i];
    k.rstd[i] = saved_rstd[c0 + i];
    k.scale[i] = gamma[c0 + i] * k.rstd[i];
    k.shift[i] = beta[c0 + i] - k.mean[i] * k.scale[i];
  }
}

// Where the ReLU mask comes from: recomputed from x, the bf16 BN output y, or the forward's mask bits (one byte per
// vector of 8 channels)
enum YKind { kMaskFromX = 0, kMaskFromY = 1, kMaskBits = 2 };

template <bool RELU, int YK>
EDL_DEVICE void masked_grad(float (&g)[8], const float (&f)[8], const bf16x8* yv, const Coef& k) {
  if (!RELU) return;
  if (YK == kMaskFromY) {
    float o[8];
    unpack8(*yv, o);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = o[i] > 0.f ? g[i] : 0.f;
  } else if (YK == kMaskBits) {
    const uint32_t b = *reinterpret_cast<const uint8_t*>(yv);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = ((b >> i) & 1u) ? g[i] : 0.f;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = fmaf(f[i], k.scale[i], k.shift[i]) > 0.f ? g[i] : 0.f;
  }
}

template <bool RELU, int YK>
__global__ void __launch_bounds__(kThreads, 1)
bn_bwd_reduce_stream_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                            const void* __restrict__ y, const float* __restrict__ gamma,
                            const float* __restrict__ beta, const float* __restrict__ saved_mean,
                            const float* __restrict__ saved_rstd, float* __restrict__ dsums, int64_t total,
                            int C) {
  extern __shared__ uint8_t smem_raw[];
  constexpr int NT = YK != kMaskFromX ? 3 : 2;
  constexpr int MT = YK == kMaskBits ? NT - 1 : -1;
  Ring<NT> r = ring_init<NT>(smem_raw);
  const int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  const int tid = threadIdx.x;
  const bool consumer = tid < kConsumers;
  const int cvecs = C / 8;
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  if (!consumer) {
    if (tid == kConsumers) {
      const void* src[NT];
      src[0] = dy;
      src[1] = x;
      if (YK != kMaskFromX) src[NT - 1] = y;
      produce<NT, MT>(r, src, total, n_chunks);
    }
  } else {
    Coef k;
    load_coef(k, saved_mean, saved_rstd, gamma, beta, (tid % cvecs) * 8);
    consume<NT, MT>(r, total, n_chunks, [&](int64_t, const bf16x8* const (&p)[NT]) {
      float g[8], f[8];
      unpack8(*p[0], g);
      unpack8(*p[1], f);
      masked_grad<RELU, YK>(g, f, p[NT - 1], k);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i] += g[i];
        acc[8 + i] = fmaf(g[i], (f[i] - k.mean[i]) * k.rstd[i], acc[8 + i]);
      }
    });
  }
  reduce_groups<16>(acc, cvecs, reinterpret_cast<float*>(r.data), consumer);
  if (consumer && tid < cvecs) {
    red_add8(&dsums[tid * 8], acc);
    red_add8(&dsums[C + tid * 8], acc + 8);
  }
}

template <bool RELU, int YK>
__global__ void __launch_bounds__(kThreads, 1)
bn_bwd_apply_stream_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                           const void* __restrict__ y, const float* __restrict__ gamma,
                           const float* __restrict__ beta, const float* __restrict__ saved_mean,
                           const float* __restrict__ saved_rstd, const float* __restrict__ dsums,
                           __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dres,
                           float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t total, int C,
                           int accumulate) {
  extern __shared__ uint8_t smem_raw[];
  constexpr int NT = YK != kMaskFromX ? 3 : 2;
  constexpr int MT = YK == kMaskBits ? NT - 1 : -1;
  Ring<NT> r = ring_init<NT>(smem_raw);
  const int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  const int tid = threadIdx.x;
  const int cvecs = C / 8;
  if (tid >= kConsumers) {
    if (tid == kConsumers) {
      const void* src[NT];
      src[0] = dy;
      src[1] = x;
      if (YK != kMaskFromX) src[NT - 1] = y;
      produce<NT, MT>(r, src, total, n_chunks);
    }
    return;
  }
  const int c0 = (tid % cvecs) * 8;
  const float inv_m = 1.f / (float)(total / C);
  Coef k;
  load_coef(k, saved_mean, saved_rstd, gamma, beta, c0);
  float k1[8], k2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float db = dsums[c0 + i], dg = dsums[C + c0 + i];
    k1[i] = db * inv_m;
    k2[i] = dg * inv_m;
    if (blockIdx.x == 0 && tid < cvecs && dgamma != nullptr) {
      if (accumulate) {
        dgamma[c0 + i] += dg;
        dbeta[c0 + i] += db;
      } else {
        dgamma[c0 + i] = dg;
        dbeta[c0 + i] = db;
      }
    }
  }
  consume<NT, MT>(r, total, n_chunks, [&](int64_t goff, const bf16x8* const (&p)[NT]) {
    float g[8], f[8];
    unpack8(*p[0], g);
    unpack8(*p[1], f);
    masked_grad<RELU, YK>(g, f, p[NT - 1], k);
    if (dres != nullptr) st_vec(dres + goff, pack8(g));
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xhat = (f[i] - k.mean[i]) * k.rstd[i];
      f[i] = k.scale[i] * (g[i] - k1[i] - xhat * k2[i]);
    }
    st_vec(dx + goff, pack8(f));
  });
}

inline int stream_grid(int64_t total) {
  int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  return (int)(n_chunks < kNumSMs ? n_chunks : kNumSMs);
}
// Reduction kernels end with 2C global reductions per CTA into the same few KB: fewer, fatter CTAs
// (a full ring of chunks each) for small tensors keep that tail short.
inline int reduce_grid(int64_t total) {
  int64_t n_chunks = (total + kChunkElems - 1) / kChunkElems;
  int64_t g = (n_chunks + kStages - 1) / kStages;
  return (int)(g < 1 ? 1 : (g < kNumSMs ? g : kNumSMs));
}

template <class K>
inline void set_smem(K kern, size_t bytes) {
  static thread_local const void* done[32];
  static thread_local int n = 0;
  for (int i = 0; i < n; ++i)
    if (done[i] == (const void*)kern) return;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  apply_carveout((const void*)kern);
  if (n < 32) done[n++] = (const void*)kern;
}

}  // namespace

#define BF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define BFW(p) reinterpret_cast<__nv_bfloat16*>(p)

bool bn_stream_supported(int64_t M, int C) {
  if (C < 8 || C > 4096 || (C & (C - 1)) != 0) return false;
  return M * C >= (int64_t)kChunkElems * 8;  // tiny tensors: the register kernels are fine
}

void bn_stats_stream(const void* x, float* sums, int64_t M, int C, cudaStream_t s) {
  const int64_t total = M * C;
  const size_t smem = ring_smem_bytes<1>() > kConsumers * 16 * 4 ? ring_smem_bytes<1>() : kConsumers * 16 * 4 + 256;
  set_smem(bn_stats_stream_kernel, smem);
  launch_pdl(bn_stats_stream_kernel, dim3(reduce_grid(total)), dim3(kThreads), smem, s, BF(x), sums, total, C);
}

bool bn_mask_supported(int64_t M, int C) { return bn_stream_supported(M, C) && C % 128 == 0; }

void bn_apply_stream(const void* x, const void* res, void* y, void* mask, const float* sums, const float* gamma,
                     const float* beta, float* running_mean, float* running_var, float* saved_mean,
                     float* saved_rstd, int64_t M, int C, float eps, float momentum, bool relu,
                     cudaStream_t s) {
  const int64_t total = M * C;
  if (res != nullptr) {
    set_smem(bn_apply_stream_kernel<true>, ring_smem_bytes<2>());
    launch_pdl(bn_apply_stream_kernel<true>, dim3(stream_grid(total)), dim3(kThreads), ring_smem_bytes<2>(), s,
        BF(x), BF(res), BFW(y), reinterpret_cast<uint8_t*>(mask), sums, gamma, beta, running_mean, running_var,
        saved_mean, saved_rstd, total, C, eps, momentum, relu ? 1 : 0);
  } else {
    set_smem(bn_apply_stream_kernel<false>, ring_smem_bytes<1>());
    launch_pdl(bn_apply_stream_kernel<false>, dim3(stream_grid(total)), dim3(kThreads), ring_smem_bytes<1>(), s,
        BF(x), (const __nv_bfloat16*)nullptr, BFW(y), (uint8_t*)nullptr, sums, gamma, beta, running_mean, running_var,
        saved_mean, saved_rstd, total, C, eps, momentum, relu ? 1 : 0);
  }
}

void bn_bwd_reduce_stream(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                          const float* beta, const float* saved_mean, const float* saved_rstd, float* dsums, int64_t M,
                          int C, bool relu, cudaStream_t s) {
  const int64_t total = M * C;
#define LAUNCH(R, Y, NT, YP)                                                                               \
  {                                                                                                        \
    set_smem(bn_bwd_reduce_stream_kernel<R, Y>, ring_smem_bytes<NT>());                                    \
    launch_pdl(bn_bwd_reduce_stream_kernel<R, Y>, dim3(reduce_grid(total)), dim3(kThreads),                \
               ring_smem_bytes<NT>(), s, BF(dy), BF(x), YP, gamma, beta, saved_mean, saved_rstd, dsums, total, C);                       \
  }
  if (!relu) LAUNCH(false, kMaskFromX, 2, y)
  else if (mask != nullptr) LAUNCH(true, kMaskBits, 3, mask)
  else if (y != nullptr) LAUNCH(true, kMaskFromY, 3, y)
  else LAUNCH(true, kMaskFromX, 2, y)
#undef LAUNCH
}

void bn_bwd_apply_stream(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                         const float* beta, const float* saved_mean, const float* saved_rstd, const float* dsums,
                         void* dx, void* dres, float* dgamma, float* dbeta, int64_t M, int C, bool relu,
                         bool accumulate, cudaStream_t s) {
  const int64_t total = M * C;
#define LAUNCH(R, Y, NT, YP)                                                                               \
  {                                                                                                        \
    set_smem(bn_bwd_apply_stream_kernel<R, Y>, ring_smem_bytes<NT>());                                     \
    launch_pdl(bn_bwd_apply_stream_kernel<R, Y>, dim3(stream_grid(total)), dim3(kThreads),                 \
               ring_smem_bytes<NT>(), s, BF(dy), BF(x), YP, gamma, beta, saved_mean, saved_rstd, dsums, BFW(dx), BFW(dres), dgamma, dbeta, \
        total, C, accumulate ? 1 : 0);                                                                     \
  }
  if (!relu) LAUNCH(false, kMaskFromX, 2, y)
  else if (mask != nullptr) LAUNCH(true, kMaskBits, 3, mask)
  else if (y != nullptr) LAUNCH(true, kMaskFromY, 3, y)
  else LAUNCH(true, kMaskFromX, 2, y)
#undef LAUNCH
}

}  // namespace edl
