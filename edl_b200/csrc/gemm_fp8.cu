// FP8 (e4m3 x e4m3 -> fp32 in registers -> bf16) GEMM for the teacher's 1x1 convolutions / classifier on
// sm_90a: wgmma.mma_async m64nNk32 .e4m3.e4m3, twice the tensor throughput of bf16 and half the
// operand bytes (SURVEY K12).  Same warp-specialised structure as gemm.cu: warp 0 TMA producer,
// warps 4..11 two consumer warpgroups that issue the MMAs of their 64 rows and then run the
// epilogue (dequantisation scale * folded-BN scale, shift, ReLU, bf16, swizzled staging, TMA store).
// A K block is 128 fp8 = one 128-byte swizzle span, so the shared-memory geometry and the operand
// descriptors are those of the bf16 kernel.  Also hosts the bf16 -> e4m3 quantisers.
//
// Two scalings share the kernel: per-tensor (one activation scale, per-output-channel weight scales, all
// folded into col_scale) and block-scaled (an fp32 scale per activation row and 128-element K block, one
// per 128x128 weight block, applied per k-block in the main loop: see Fp8BlockParams).
//
// Block-scaled epilogue variants (compile-time EPI argument, default plain), for the sequence teacher's linear layers:
// kEpiAdd adds a bf16 residual tile, TMA-loaded by the producer warp while the main loop runs, after the bias;
// kEpiGeluQ applies bias + erf-GELU, rounds to bf16 and quantises each row's 128 columns to e4m3 with their own block
// scale, writing the next GEMM's A operand and its sa directly (the rules of quantize_e4m3_blocks).
#include <cuda.h>
#include <cuda_fp8.h>
#include <cstdint>
#include <cstdio>
#include <type_traits>

#include "gemm.h"
#include "kernels.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kBlockM = 128;
constexpr int kBlockKBytes = 128;   // = 128 e4m3 elements
constexpr int kMmaKBytes = 32;
constexpr int kThreads = 384;   // producer warpgroup (one warp works) + two consumer warpgroups

struct Fp8Params {
  int M, N, K;
  const float* col_scale;
  const float* col_shift;
  int relu;
};

// Block-scaled variant: sa fp32 [KB, M] (one scale per row and 128-element K block, K-block-major so that a
// k-block's scales for a tile's rows are contiguous), sb fp32 [ceil(N/128), KB] (one per 128x128 weight block).
struct Fp8BlockParams : Fp8Params {
  const float* sa;
  const float* sb;
};

// kEpiGeluQ: the output's block scales, fp32 [ceil(N/128), M] (the sa layout of the GEMM it feeds)
struct Fp8BlockQParams : Fp8BlockParams {
  float* sa_out;
};

constexpr int kEpiPlain = 0, kEpiAdd = 1, kEpiGeluQ = 2;

// ADD: a second tile-sized region after the ring holds the residual tile (kEpiAdd)
template <int BLOCK_N, int STAGES, bool ADD = false>
struct Smem {
  static constexpr int kABytes = kBlockM * kBlockKBytes;
  static constexpr int kBBytes = BLOCK_N * kBlockKBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kDBytes = kBlockM * BLOCK_N * 2;
  static constexpr int kTileBytes = STAGES * kStageBytes > kDBytes ? STAGES * kStageBytes : kDBytes;
  static constexpr int kAddOffset = kTileBytes;
  static constexpr int kBarOffset = kTileBytes + (ADD ? kDBytes : 0);
  static constexpr int kTotal = kBarOffset + 256 + 1024;
};

template <int BLOCK_N, int STAGES, typename P, int EPI = kEpiPlain>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const __grid_constant__ CUtensorMap tmD, const P p, const __grid_constant__ CUtensorMap tmAdd) {
  constexpr bool kBlockScaled = std::is_base_of<Fp8BlockParams, P>::value;
  static_assert(EPI == kEpiPlain || kBlockScaled, "epilogue variants are block-scaled only");
  static_assert(EPI != kEpiGeluQ || BLOCK_N == 128, "kEpiGeluQ: a tile's columns are one 128-element scale block");
  using L = Smem<BLOCK_N, STAGES, EPI == kEpiAdd>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  [[maybe_unused]] uint64_t* add_bar = empty_bar + STAGES;   // kEpiAdd: the residual tile landed
  [[maybe_unused]] uint8_t* sadd = smem + L::kAddOffset;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int m0 = (blockIdx.x / tiles_n) * kBlockM;
  const int n0 = (blockIdx.x % tiles_n) * BLOCK_N;
  const int num_kb = (p.K + kBlockKBytes - 1) / kBlockKBytes;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    ptx::prefetch_tmap(&tmD);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    if constexpr (EPI == kEpiAdd) {
      ptx::prefetch_tmap(&tmAdd);
      ptx::mbar_init(add_bar, 1);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if constexpr (EPI == kEpiAdd) {
      // the residual tile goes to its own region first, so its load hides behind the whole main loop; the 64-column
      // halves past N are not loaded (rows past M are zero-filled by the TMA unit)
      uint32_t halves = 0;
#pragma unroll
      for (int h = 0; h < (BLOCK_N + 63) / 64; ++h) halves += (n0 + h * 64 < p.N) ? 1u : 0u;
      if (ptx::elect_one()) {
        ptx::mbar_arrive_expect_tx(add_bar, halves * (kBlockM * 128));
#pragma unroll
        for (int h = 0; h < (BLOCK_N + 63) / 64; ++h)
          if (n0 + h * 64 < p.N) ptx::tma_load_2d(sadd + h * (kBlockM * 128), &tmAdd, add_bar, n0 + h * 64, m0);
      }
      __syncwarp();
    }
    // warp-uniform loops, one elected lane issues (see gemm_persist.cu)
    for (int i = 0; i < num_kb; ++i) {
      const int s = i % STAGES;
      const uint32_t ph = (i / STAGES) & 1;
      ptx::mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* sa = smem + s * L::kStageBytes;
      if (ptx::elect_one()) {
        ptx::mbar_arrive_expect_tx(&full_bar[s], L::kStageBytes);
        ptx::tma_load_2d(sa, &tmA, &full_bar[s], i * kBlockKBytes, m0);
        ptx::tma_load_2d(sa + L::kABytes, &tmB, &full_bar[s], i * kBlockKBytes, n0);
      }
      __syncwarp();
    }
  } else if (warp >= 4) {
    // consumers (warps 4..11): each warpgroup owns 64 rows of the tile, MMA then epilogue
    const int cw = (warp - 4) >> 2;
    const int et = threadIdx.x - 128;
    const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // first accumulator row of this thread (second: + 8)
    const int cq = (lane & 3) * 2;
    float acc[BLOCK_N / 2];
    if constexpr (kBlockScaled) {
      // Per k-block: the 4 MMAs go into tmp (scale-d = 0 on the first), then tmp is promoted into acc with
      // this block's row scale * weight-block scale.  The scale loads are issued before the full-barrier wait
      // and first read after the MMAs, so their latency hides behind both.  Rows past M read scale 0 (their
      // stores are clipped); a tile's BLOCK_N <= 128 columns lie in one 128-row weight block.
      float tmp[BLOCK_N / 2];
#pragma unroll
      for (int j = 0; j < BLOCK_N / 2; ++j) acc[j] = 0.f;
      const int r0 = m0 + row, r1 = m0 + row + 8;
      const float* sb_tile = p.sb + (size_t)(n0 / 128) * num_kb;
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        const float* sa_kb = p.sa + (size_t)i * p.M;
        const float sbk = __ldg(sb_tile + i);
        const float sa0 = r0 < p.M ? __ldg(sa_kb + r0) : 0.f;
        const float sa1 = r1 < p.M ? __ldg(sa_kb + r1) : 0.f;
        ptx::mbar_wait(&full_bar[s], (i / STAGES) & 1);
        const uint32_t sa = ptx::smem_u32(smem + s * L::kStageBytes);
        const uint64_t da0 = ptx::make_smem_desc(sa + cw * 8192, 16, 1024);
        const uint64_t db0 = ptx::make_smem_desc(sa + L::kABytes, 16, 1024);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockKBytes / kMmaKBytes; ++k)
          ptx::WgmmaE4m3<BLOCK_N>::mma(tmp, da0 + (uint64_t)(k * (kMmaKBytes >> 4)), db0 + (uint64_t)(k * (kMmaKBytes >> 4)),
                                       k != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[s]);
        const float f0 = sa0 * sbk, f1 = sa1 * sbk;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          acc[4 * j] = fmaf(tmp[4 * j], f0, acc[4 * j]);
          acc[4 * j + 1] = fmaf(tmp[4 * j + 1], f0, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(tmp[4 * j + 2], f1, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(tmp[4 * j + 3], f1, acc[4 * j + 3]);
        }
      }
    } else {
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        ptx::mbar_wait(&full_bar[s], (i / STAGES) & 1);
        const uint32_t sa = ptx::smem_u32(smem + s * L::kStageBytes);
        const uint64_t da0 = ptx::make_smem_desc(sa + cw * 8192, 16, 1024);
        const uint64_t db0 = ptx::make_smem_desc(sa + L::kABytes, 16, 1024);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockKBytes / kMmaKBytes; ++k)     // start-address field counts 16-byte units
          ptx::WgmmaE4m3<BLOCK_N>::mma(acc, da0 + (uint64_t)(k * (kMmaKBytes >> 4)), db0 + (uint64_t)(k * (kMmaKBytes >> 4)),
                                       (i | k) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
        if (i > 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[(i - 1) % STAGES]);
      }
      ptx::wgmma_wait<0>();
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");       // the ring is drained: it becomes the staging tile
    uint8_t* sd = smem;
    if constexpr (EPI == kEpiGeluQ) {
      // g = bf16(gelu(acc + bias)) in place of acc; this thread's two rows' max|g| over its 32 columns, then over the
      // lane quad that holds the row's other 96 (columns past N are 0: B is zero-filled and the bias read guarded)
      float amax0 = 0.f, amax1 = 0.f;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + j * 8 + cq;
        const float sh0 = (p.col_shift != nullptr && col < p.N) ? __ldg(p.col_shift + col) : 0.f;
        const float sh1 = (p.col_shift != nullptr && col + 1 < p.N) ? __ldg(p.col_shift + col + 1) : 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float v = acc[4 * j + e] + ((e & 1) ? sh1 : sh0);
          acc[4 * j + e] = __bfloat162float(__float2bfloat16_rn(0.5f * v * (1.f + erff(v * 0.70710678118654752f))));
        }
        amax0 = fmaxf(amax0, fmaxf(fabsf(acc[4 * j]), fabsf(acc[4 * j + 1])));
        amax1 = fmaxf(amax1, fmaxf(fabsf(acc[4 * j + 2]), fabsf(acc[4 * j + 3])));
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        amax0 = fmaxf(amax0, __shfl_xor_sync(0xffffffffu, amax0, o));
        amax1 = fmaxf(amax1, __shfl_xor_sync(0xffffffffu, amax1, o));
      }
      const float s0 = amax0 > 0.f ? __fdiv_rn(amax0, 448.f) : 1.f;
      const float s1 = amax1 > 0.f ? __fdiv_rn(amax1, 448.f) : 1.f;
      if (cq == 0) {
        float* so = p.sa_out + (size_t)(n0 / 128) * p.M + m0;
        if (m0 + row < p.M) so[row] = s0;
        if (m0 + row + 8 < p.M) so[row + 8] = s1;
      }
      // e4m3 bytes into a 128 x 128-byte staging tile, 128-byte swizzle (16-byte chunk c of row r at c ^ (r & 7))
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int off = (j & 1) * 8 + cq;
        const __nv_fp8x2_storage_t q0 = __nv_cvt_float2_to_fp8x2(
            make_float2(__fdiv_rn(acc[4 * j], s0), __fdiv_rn(acc[4 * j + 1], s0)), __NV_SATFINITE, __NV_E4M3);
        const __nv_fp8x2_storage_t q1 = __nv_cvt_float2_to_fp8x2(
            make_float2(__fdiv_rn(acc[4 * j + 2], s1), __fdiv_rn(acc[4 * j + 3], s1)), __NV_SATFINITE, __NV_E4M3);
        *reinterpret_cast<__nv_fp8x2_storage_t*>(sd + row * 128 + (((j >> 1) ^ (row & 7)) << 4) + off) = q0;
        *reinterpret_cast<__nv_fp8x2_storage_t*>(sd + (row + 8) * 128 + (((j >> 1) ^ ((row + 8) & 7)) << 4) + off) = q1;
      }
      ptx::fence_proxy_async_smem();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (et == 0) {
        ptx::tma_store_2d(&tmD, sd, n0, m0);              // clipped at M and N
        ptx::tma_store_commit();
        ptx::tma_store_wait_read0();
      }
    } else {
      if constexpr (EPI == kEpiAdd) ptx::mbar_wait(add_bar, 0);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + j * 8 + cq;
        const float sc0 = (p.col_scale != nullptr && col < p.N) ? p.col_scale[col] : 1.f;
        const float sc1 = (p.col_scale != nullptr && col + 1 < p.N) ? p.col_scale[col + 1] : 1.f;
        const float sh0 = (p.col_shift != nullptr && col < p.N) ? p.col_shift[col] : 0.f;
        const float sh1 = (p.col_shift != nullptr && col + 1 < p.N) ? p.col_shift[col + 1] : 0.f;
        float v0 = fmaf(acc[4 * j], sc0, sh0), v1 = fmaf(acc[4 * j + 1], sc1, sh1);
        float v2 = fmaf(acc[4 * j + 2], sc0, sh0), v3 = fmaf(acc[4 * j + 3], sc1, sh1);
        if constexpr (EPI == kEpiAdd) {
          // the residual tile has the staging tile's swizzled layout: read each value where it will be stored
          const uint8_t* ap = sadd + (j >> 3) * (kBlockM * 128) + cq * 2;
          const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ap + row * 128 + (((j & 7) ^ (row & 7)) << 4)));
          const float2 a1 = __bfloat1622float2(
              *reinterpret_cast<const __nv_bfloat162*>(ap + (row + 8) * 128 + (((j & 7) ^ ((row + 8) & 7)) << 4)));
          v0 += a0.x; v1 += a0.y; v2 += a1.x; v3 += a1.y;
        }
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
        uint8_t* hp = sd + (j >> 3) * (kBlockM * 128) + cq * 2;
        *reinterpret_cast<__nv_bfloat162*>(hp + row * 128 + (((j & 7) ^ (row & 7)) << 4)) = __floats2bfloat162_rn(v0, v1);
        *reinterpret_cast<__nv_bfloat162*>(hp + (row + 8) * 128 + (((j & 7) ^ ((row + 8) & 7)) << 4)) = __floats2bfloat162_rn(v2, v3);
      }
      ptx::fence_proxy_async_smem();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (et == 0) {
#pragma unroll
        for (int h = 0; h < (BLOCK_N + 63) / 64; ++h)
          if (n0 + h * 64 < p.N) ptx::tma_store_2d(&tmD, sd + h * (kBlockM * 128), n0 + h * 64, m0);
        ptx::tma_store_commit();
        ptx::tma_store_wait_read0();
      }
    }
  }
}

template <int BLOCK_N, int STAGES, typename P, int EPI = kEpiPlain>
const char* launch(const GemmFp8Args& g, cudaStream_t stream) {
  using L = Smem<BLOCK_N, STAGES, EPI == kEpiAdd>;
  alignas(64) CUtensorMap tmA, tmB, tmD, tmAdd{};
  {
    const uint64_t dims[2] = {(uint64_t)g.K, (uint64_t)g.M};
    const uint64_t st[1] = {(uint64_t)g.lda};
    const uint32_t box[2] = {kBlockKBytes, kBlockM};
    if (const char* e = encode_tmap(&tmA, g.A, 2, dims, st, box, 1)) return e;
  }
  {
    const uint64_t dims[2] = {(uint64_t)g.K, (uint64_t)g.N};
    const uint64_t st[1] = {(uint64_t)g.ldb};
    const uint32_t box[2] = {kBlockKBytes, (uint32_t)BLOCK_N};
    if (const char* e = encode_tmap(&tmB, g.B, 2, dims, st, box, 1)) return e;
  }
  if constexpr (EPI == kEpiGeluQ) {           // e4m3 bytes: one 128-byte box row = the tile's 128 columns
    const uint64_t dims[2] = {(uint64_t)g.N, (uint64_t)g.M};
    const uint64_t st[1] = {(uint64_t)g.ldd};
    const uint32_t box[2] = {128, kBlockM};
    if (const char* e = encode_tmap(&tmD, g.D, 2, dims, st, box, 1)) return e;
  } else {
    const uint64_t dims[2] = {(uint64_t)g.N, (uint64_t)g.M};
    const uint64_t st[1] = {(uint64_t)g.ldd * 2};
    const uint32_t box[2] = {64, kBlockM};
    if (const char* e = encode_tmap(&tmD, g.D, 2, dims, st, box, 2)) return e;
  }
  if constexpr (EPI == kEpiAdd) {
    const uint64_t dims[2] = {(uint64_t)g.N, (uint64_t)g.M};
    const uint64_t st[1] = {(uint64_t)g.ld_add * 2};
    const uint32_t box[2] = {64, kBlockM};
    if (const char* e = encode_tmap(&tmAdd, g.add, 2, dims, st, box, 2)) return e;
  }
  auto kern = gemm_fp8_wgmma_kernel<BLOCK_N, STAGES, P, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  P p{};
  p.M = g.M;
  p.N = g.N;
  p.K = g.K;
  p.col_scale = g.col_scale;
  p.col_shift = g.col_shift;
  p.relu = g.relu ? 1 : 0;
  if constexpr (std::is_base_of<Fp8BlockParams, P>::value) {
    p.sa = g.a_scales;
    p.sb = g.b_scales;
  }
  if constexpr (std::is_same<P, Fp8BlockQParams>::value) p.sa_out = g.a_scales_out;
  const int tiles = ((g.M + kBlockM - 1) / kBlockM) * ((g.N + BLOCK_N - 1) / BLOCK_N);
  kern<<<tiles, kThreads, L::kTotal, stream>>>(tmA, tmB, tmD, p, tmAdd);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

__global__ void __launch_bounds__(256)
quantize_e4m3_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, int64_t n,
                     const float* __restrict__ scale, float* __restrict__ amax_out) {
  const float sc = *scale;   // q = sat(x / scale) with a true division: x * (1 / scale) rounds some ties the other way
  float amax = 0.f;
  const int64_t nvec = n / 8;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const bf16x8 v = ld_vec(x + i * 8);
    float f[8];
    unpack8(v, f);
    uint8_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      amax = fmaxf(amax, fabsf(f[j]));
      o[j] = (uint8_t)__nv_cvt_float_to_fp8(__fdiv_rn(f[j], sc), __NV_SATFINITE, __NV_E4M3);
    }
    *reinterpret_cast<uint2*>(q + i * 8) = *reinterpret_cast<const uint2*>(o);
  }
  if (blockIdx.x == 0)
    for (int64_t i = nvec * 8 + threadIdx.x; i < n; i += blockDim.x) {
      const float f = __bfloat162float(x[i]);
      amax = fmaxf(amax, fabsf(f));
      q[i] = (uint8_t)__nv_cvt_float_to_fp8(__fdiv_rn(f, sc), __NV_SATFINITE, __NV_E4M3);
    }
  if (amax_out != nullptr) {
    amax = warp_max(amax);
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax_out), __float_as_int(amax));  // amax >= 0
  }
}

// Row-block quantiser: one half-warp per (row m, 128-element K block b).  Each lane loads 8 bf16 (16 bytes),
// the block's max|x| is reduced with shuffles across the 16 lanes that share it, s = amax / 448 (1 for an
// all-zero block) goes to sa[b, m], and every lane stores its 8 bytes sat(x / s).  K % 8 == 0, so a lane's
// 8 elements are either all inside the (possibly shorter) tail block or all past K.
__global__ void __launch_bounds__(256)
quantize_e4m3_blocks_kernel(const __nv_bfloat16* __restrict__ x, int64_t lda, uint8_t* __restrict__ q,
                            float* __restrict__ sa, int M, int K) {
  const int kbs = (K + kBlockKBytes - 1) / kBlockKBytes;
  const int segs = M * kbs;
  const int hl = threadIdx.x & 15;
  const unsigned mask = 0xffffu << (threadIdx.x & 16);   // the 16 lanes of this half-warp
  for (int seg = blockIdx.x * 16 + (threadIdx.x >> 4); seg < segs; seg += gridDim.x * 16) {
    const int m = seg / kbs, b = seg - m * kbs;
    const int k = b * kBlockKBytes + hl * 8;
    const bool live = k < K;
    float f[8];
    if (live) {
      unpack8(ld_vec(x + (int64_t)m * lda + k), f);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(f[j]));
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(mask, amax, o));
    const float s = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
    if (hl == 0) sa[(int64_t)b * M + m] = s;
    if (live) {
      uint8_t o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        o[j] = (uint8_t)__nv_cvt_float_to_fp8(__fdiv_rn(f[j], s), __NV_SATFINITE, __NV_E4M3);
      *reinterpret_cast<uint2*>(q + (int64_t)m * K + k) = *reinterpret_cast<const uint2*>(o);
    }
  }
}

const char* check_fp8_args(const GemmFp8Args& g) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return "empty GEMM";
  if (g.K % 16 != 0 || g.lda % 16 != 0 || g.ldb % 16 != 0 || g.ldd % 8 != 0) return "fp8 GEMM needs 16-byte aligned rows";
  if (g.device >= 0) {
    cudaError_t e = cudaSetDevice(g.device);
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  return nullptr;
}

}  // namespace

const char* gemm_fp8(const GemmFp8Args& g, cudaStream_t stream) {
  if (const char* e = check_fp8_args(g)) return e;
  return g.N <= 64 ? launch<64, 4, Fp8Params>(g, stream) : launch<128, 3, Fp8Params>(g, stream);
}

const char* gemm_fp8_blockscaled(const GemmFp8Args& g, cudaStream_t stream) {
  if (g.a_scales == nullptr || g.b_scales == nullptr) return "block-scaled fp8 GEMM needs both scale tensors";
  if (const char* e = check_fp8_args(g)) return e;
  if (g.add != nullptr) {
    if (g.N % 8 != 0 || g.ld_add % 8 != 0 || (reinterpret_cast<uintptr_t>(g.add) & 15) != 0)
      return "fp8 GEMM addend needs 16-byte aligned rows";
    // one tile per CTA: 64-column tiles when they need fewer waves of 64-column work than 128-column tiles do
    // (small M; T = 2330 tokens at N = 768 is 114 tiles of 128 x 128, one wave either way)
    const int mt = (g.M + kBlockM - 1) / kBlockM;
    const int w128 = 2 * ((mt * ((g.N + 127) / 128) + kNumSMs - 1) / kNumSMs);
    const int w64 = (mt * ((g.N + 63) / 64) + kNumSMs - 1) / kNumSMs;
    return (g.N <= 64 || w64 < w128) ? launch<64, 4, Fp8BlockParams, kEpiAdd>(g, stream)
                                     : launch<128, 3, Fp8BlockParams, kEpiAdd>(g, stream);
  }
  return g.N <= 64 ? launch<64, 4, Fp8BlockParams>(g, stream) : launch<128, 3, Fp8BlockParams>(g, stream);
}

const char* gemm_fp8_blockscaled_gelu_e4m3(const GemmFp8Args& g, cudaStream_t stream) {
  if (g.a_scales == nullptr || g.b_scales == nullptr || g.a_scales_out == nullptr)
    return "block-scaled fp8 GEMM needs both scale tensors and the output scales";
  if (g.col_scale != nullptr || g.relu || g.add != nullptr) return "GELU e4m3 epilogue: bias only";
  if (const char* e = check_fp8_args(g)) return e;
  if (g.N % 16 != 0 || g.ldd % 16 != 0) return "GELU e4m3 epilogue needs 16-byte aligned output rows";
  return launch<128, 3, Fp8BlockQParams, kEpiGeluQ>(g, stream);
}

const char* quantize_e4m3_blocks(const void* x, int64_t lda, void* q, float* sa, int M, int K, cudaStream_t s) {
  if (M <= 0 || K <= 0) return "empty input";
  if (K % 8 != 0 || lda % 8 != 0) return "block quantiser needs 16-byte aligned rows";
  const int64_t segs = (int64_t)M * ((K + kBlockKBytes - 1) / kBlockKBytes);
  if (segs > INT32_MAX / 2) return "block quantiser: too many blocks";
  int64_t blocks = (segs + 15) / 16;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  quantize_e4m3_blocks_kernel<<<(int)blocks, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), lda,
                                                          reinterpret_cast<uint8_t*>(q), sa, M, K);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

void quantize_e4m3(const void* x, void* q, int64_t n, const float* scale, float* amax_out, cudaStream_t s) {
  int64_t blocks = (n / 8 + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  if (blocks < 1) blocks = 1;
  quantize_e4m3_kernel<<<(int)blocks, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                    reinterpret_cast<uint8_t*>(q), n, scale, amax_out);
}

}  // namespace edl
