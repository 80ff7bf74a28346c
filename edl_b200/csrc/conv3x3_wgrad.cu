// Weight gradient of the 3x3 / stride 1 / pad 1 NHWC convolution on wgmma (SURVEY K1, wgrad third).
// The reference gets it from cuDNN through Paddle's conv2d_grad (example/distill/resnet/models/
// resnet_vd.py:153-162).
//
//   dW[co, r, s, ci] = sum over pixels (n, h, w) of  dY[n, h, w, co] * X[n, h + r - 1, w + s - 1, ci]
//
// As a GEMM per filter tap: M = Cout, N = Cin, K = pixels, both operands "MN-major" (the channel dimension is
// the contiguous one in NHWC, the reduction runs over pixels):
//   A tile = 4-D TMA box {64 ch, W, BH, NB} of dY          -> smem [KB pixel rows][64 ch = 128 B], 128B swizzle
//   B tile = the SAME box of X shifted by (s - 1, r - 1)    -> out-of-image pixels are zero-filled by the TMA
//                                                              unit (= the padding; no im2col, no index math)
// One CTA owns a 128 (Cout) x 64 (Cin) tile of ONE FILTER ROW r: the dY tile of a pixel block is loaded once
// and multiplied with the three shifted X tiles (s = 0, 1, 2) into three register accumulators, so dY crosses
// L2 -> SM once per row instead of once per tap.  Without a split of the pixel reduction the CTA writes its tile as
// bf16 straight into the flat gradient bucket (+= when accumulating); split over gridDim.z CTAs, every CTA stores its
// fp32 partial tile and splitk_reduce sums them into the bucket -- the same scheme as the 1x1 wgrad GEMM (gemm.cu).
//
//   warp 0      : TMA producer (2 + 3 box loads per pixel block into a 3-stage ring)
//   warps 4..11 : two consumer warpgroups, one per 64-channel chunk of dY: wgmma.mma_async into three 64 x 64 fp32
//                 register accumulators (one per tap), then the epilogue (smem staging -> bf16 or partial-tile stores)
#include <cuda.h>

#include "gemm.h"
#include "kernels.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kBlockM = 128;      // Cout rows per tile
constexpr int kBlockN = 64;       // Cin columns per tile (one 128-byte swizzle span)
constexpr int kMaxKB = 112;       // pixel rows per K block (multiple of 16; 112 = 2x56 = 4x28 = 8x14 = 16x7)
constexpr int kMmaK = 16;
constexpr int kStages = 3;
constexpr int kThreads = 384;          // producer warpgroup (one warp works) + two consumer warpgroups
constexpr int kEpiThreads = 256;
constexpr int kChunkBytes = kMaxKB * 128;                 // one [KB][64 ch] operand chunk (stride in the ring)
constexpr int kStageBytes = (2 + 3) * kChunkBytes;        // A: 2 chunks of 64 Cout; B: 3 taps x 64 Cin
constexpr int kBarOffset = kStages * kStageBytes;
constexpr int kSmemTotal = kBarOffset + 256 + 1024;
constexpr int kPitch = kBlockN * 4 + 16;                  // fp32 staging row pitch (bytes)
constexpr int kVecPerRow = kBlockN / 4;

struct WgradParams {
  int Cout, Cin;
  int BH, NB, HB;            // box rows / images, row blocks per image
  int KB;                    // pixel rows per block = W * BH * NB (multiple of 16, <= kMaxKB)
  int total_kb, kb_per_split;
  int tiles_n;
  __nv_bfloat16* out;        // bf16 [Cout][9*Cin] (KRSC)
  int accumulate;
  int stride;                // 1, or 2: X rows 2*h + r - 1 (the columns are subsampled by the tensor map)
  float* part;               // split-K partial tiles [split][ctas][128 x TAPS*64] (gridDim.z > 1)
};

// TAPS = filter taps per CTA: 3 (one filter row of the 3x3 convolution; out is KRSC [Cout][9*Cin]), or 1 (the 1x1 / pad 0 /
// stride 2 convolution: X pixel (2h, 2w) only, one accumulator, out is [Cout][Cin]).
template <int TAPS>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                     const WgradParams p) {
  static_assert(TAPS == 3 || TAPS == 1, "a filter row of the 3x3, or the 1x1 centre tap");
  constexpr int kRows = TAPS == 3 ? 3 : 1;      // filter rows, one CTA each
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // blockIdx.x = (tile * kRows + r); tile = mt * tiles_n + nt
  const int r = blockIdx.x % kRows;
  const int tile = blockIdx.x / kRows;
  const int m0 = (tile / p.tiles_n) * kBlockM;
  const int n0 = (tile % p.tiles_n) * kBlockN;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  int kb_end = kb_begin + p.kb_per_split;
  if (kb_end > p.total_kb) kb_end = p.total_kb;
  const int num_kb = kb_end - kb_begin;
  const bool two_chunks = m0 + 64 < p.Cout;     // Cout == 64: rows 64..127 of the accumulators are never stored
  const uint32_t chunk_tx = (uint32_t)p.KB * 128u;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmDy);
    ptx::prefetch_tmap(&tmX);
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (num_kb > 0) {
    if (warp == 0) {
      // ------------------------------------------------------------ TMA producer
      // warp-uniform loop, one elected lane issues (gemm_persist.cu explains why not `if (lane == 0)` around the loop)
      for (int i = 0; i < num_kb; ++i) {
        const int st = i % kStages;
        const uint32_t ph = (i / kStages) & 1;
        ptx::mbar_wait(&empty_bar[st], ph ^ 1);
        uint8_t* sa = smem + st * kStageBytes;
        uint8_t* sb = sa + 2 * kChunkBytes;
        const int kb = kb_begin + i;
        const int h0 = (kb % p.HB) * p.BH;
        const int img0 = (kb / p.HB) * p.NB;
        if (ptx::elect_one()) {
          ptx::mbar_arrive_expect_tx(&full_bar[st], chunk_tx * (two_chunks ? 2u + TAPS : 1u + TAPS));
          ptx::tma_load_4d(sa, &tmDy, &full_bar[st], m0, 0, h0, img0);
          if (two_chunks) ptx::tma_load_4d(sa + kChunkBytes, &tmDy, &full_bar[st], m0 + 64, 0, h0, img0);
#pragma unroll
          for (int s = 0; s < TAPS; ++s)
            ptx::tma_load_4d(sb + s * kChunkBytes, &tmX, &full_bar[st], n0, TAPS == 3 ? s - 1 : 0,
                             h0 * p.stride + (TAPS == 3 ? r - 1 : 0), img0);
        }
        __syncwarp();
      }
    } else if (warp >= 4) {
      // ------------------------------------------------------------ consumers: MMA, then epilogue (warps 4..11)
      const int cw = (warp - 4) >> 2;                            // consumer warpgroup = 64-channel chunk of dY
      const int et = threadIdx.x - 128;
      const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // first accumulator row of this thread (second: + 8)
      const int cq = (lane & 3) * 2;
      float acc[TAPS][kBlockN / 2];
      using Mma = ptx::WgmmaBf16<kBlockN, 1, 1>;
      const int ksteps = p.KB / kMmaK;
      for (int i = 0; i < num_kb; ++i) {
        const int st = i % kStages;
        ptx::mbar_wait(&full_bar[st], (i / kStages) & 1);
        const uint32_t sa = ptx::smem_u32(smem + st * kStageBytes) + cw * kChunkBytes;
        const uint32_t sb = ptx::smem_u32(smem + st * kStageBytes) + 2 * kChunkBytes;
        // MN-major, 128B swizzle: 16 pixel rows = 2048 B per k step (128 in the descriptor's 16-byte units),
        // 8-row groups 1024 B apart
        const uint64_t da0 = ptx::make_smem_desc(sa, kChunkBytes, 1024);
        const uint64_t db0 = ptx::make_smem_desc(sb, kChunkBytes, 1024);
        ptx::wgmma_fence();
        for (int k = 0; k < ksteps; ++k) {
#pragma unroll
          for (int s = 0; s < TAPS; ++s)
            Mma::mma(acc[s], da0 + (uint64_t)(k * 128), db0 + (uint64_t)(s * (kChunkBytes >> 4) + k * 128),
                     (i | k) != 0 ? 1u : 0u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[st]);
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");   // both groups are done reading the ring
      uint8_t* sf = smem;                        // the ring is drained: fp32 staging tile
      int rows_valid = p.Cout - m0;
      if (rows_valid > kBlockM) rows_valid = kBlockM;
      const int64_t ldw = (int64_t)(TAPS * TAPS) * p.Cin;
      const bool direct = gridDim.z == 1;
#pragma unroll
      for (int s = 0; s < TAPS; ++s) {
#pragma unroll
        for (int j = 0; j < kBlockN / 8; ++j) {
          *reinterpret_cast<float2*>(sf + row * kPitch + (j * 8 + cq) * 4) = make_float2(acc[s][4 * j], acc[s][4 * j + 1]);
          *reinterpret_cast<float2*>(sf + (row + 8) * kPitch + (j * 8 + cq) * 4) = make_float2(acc[s][4 * j + 2], acc[s][4 * j + 3]);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int64_t col0 = TAPS == 3 ? (int64_t)(r * 3 + s) * p.Cin + n0 : (int64_t)n0;
#pragma unroll 1   // one 16-byte piece per iteration, as in version 2 below
        for (int f = et; f < rows_valid * kVecPerRow; f += kEpiThreads) {
          const int rr = f / kVecPerRow, c4 = (f % kVecPerRow) * 4;
          const float4 t = *reinterpret_cast<const float4*>(sf + rr * kPitch + c4 * 4);
          if (direct) {
            // this CTA saw every pixel: bf16 (+= bucket) straight from the staged tile
            store_bf16x4(p.out + (int64_t)(m0 + rr) * ldw + col0 + c4, t, p.accumulate);
          } else {
            *reinterpret_cast<float4*>(p.part + ((int64_t)blockIdx.z * gridDim.x + blockIdx.x) * (kBlockM * TAPS * kBlockN) +
                                       rr * (TAPS * kBlockN) + s * kBlockN + c4) = t;
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // staging tile is reused by the next tap
      }
    }
  }
}

// =====================================================================================================
// Version 2: ONE X load per (pixel block, filter row) serves the three taps s = 0, 1, 2.
//
// Version 1 above needs 5 operand chunks per pixel block for 21 MMAs.
// Here both operands are loaded as boxes {64 ch, Wb, BH, NB} that START AT COLUMN w = -1 (Wb >= W + 1): the TMA
// unit zero-fills column -1 (and everything right of the image), so every image row is followed by at least one
// zero pixel.  In shared memory the pixel rows (K index) of both tiles are 128 B apart, and the X pixel a tap
// (r, s) needs for the dY pixel at K row k sits at K row k + (s - 1) of the SAME X tile: the three taps are the
// same tile read through descriptors whose start address is shifted by -128 / 0 / +128 bytes.  Where the shift
// crosses an image row it lands on a zero pixel of one of the operands (dY's column -1 / X's column -1); the rows
// just outside the tile are zeroed once at kernel start.  Per pixel block: 2 dY chunks + BLOCK_N/64 X chunks
// for 3 * KB/16 MMAs of N = BLOCK_N -- with BLOCK_N = 128 that is 2.6x fewer bytes per FLOP than version 1.
constexpr int kMaxKB2 = 128;
constexpr int kChunkA2 = kMaxKB2 * 128;                    // 16 KB per 64-channel dY chunk
constexpr int kPad2 = 1024;                                // zero rows before / after an X tile (8 rows)
constexpr int kChunkB2 = kChunkA2 + 2 * kPad2;
constexpr int kStages2 = 3;

template <int BLOCK_N>
struct W2Smem {
  static constexpr int kNCh = BLOCK_N / 64;
  static constexpr int kStage = 2 * kChunkA2 + kNCh * kChunkB2;
  static constexpr int kBar = kStages2 * kStage;
  static constexpr int kTotal = kBar + 256 + 1024;
  static constexpr int kPitch = BLOCK_N * 4 + 16;
  static_assert(128 * kPitch <= kBar, "fp32 staging tile must fit in the drained ring");
};

struct Wgrad2Params {
  int Cout, Cin;
  int BH, NB, HB, KB;
  int total_kb, kb_per_split;
  int tiles_n;
  int base_offset_mode;      // 0: descriptor base offset 0 (address-based swizzle); 1: (addr >> 7) & 7
  __nv_bfloat16* out;
  int accumulate;
  float* part;               // split-K partial tiles [split][ctas][128 x 3*BLOCK_N] (gridDim.z > 1)
};

template <int BLOCK_N>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_wgrad2_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                      const Wgrad2Params p) {
  using L = W2Smem<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBar);
  uint64_t* empty_bar = full_bar + kStages2;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x % 3;
  const int tile = blockIdx.x / 3;
  const int m0 = (tile / p.tiles_n) * kBlockM;
  const int n0 = (tile % p.tiles_n) * BLOCK_N;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  int kb_end = kb_begin + p.kb_per_split;
  if (kb_end > p.total_kb) kb_end = p.total_kb;
  const int num_kb = kb_end - kb_begin;
  const bool two_chunks = m0 + 64 < p.Cout;
  const uint32_t chunk_tx = (uint32_t)p.KB * 128u;

  // the X regions of the ring are zeroed ONCE: the TMA only ever writes rows [0, KB) of a tile, the rows around it
  // (read by the shifted descriptors at the first / last K row) stay zero for the whole kernel
  for (int s = 0; s < kStages2; ++s) {
    uint4* zb = reinterpret_cast<uint4*>(smem + s * L::kStage + 2 * kChunkA2);
    for (int i = threadIdx.x; i < L::kNCh * kChunkB2 / 16; i += kThreads) zb[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  ptx::fence_proxy_async_smem();
  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmDy);
    ptx::prefetch_tmap(&tmX);
    for (int s = 0; s < kStages2; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (num_kb > 0) {
    if (warp == 0) {
      for (int i = 0; i < num_kb; ++i) {
        const int st = i % kStages2;
        const uint32_t ph = (i / kStages2) & 1;
        ptx::mbar_wait(&empty_bar[st], ph ^ 1);
        uint8_t* sa = smem + st * L::kStage;
        uint8_t* sb = sa + 2 * kChunkA2;
        const int kb = kb_begin + i;
        const int h0 = (kb % p.HB) * p.BH;
        const int img0 = (kb / p.HB) * p.NB;
        if (ptx::elect_one()) {
          ptx::mbar_arrive_expect_tx(&full_bar[st], chunk_tx * (uint32_t)((two_chunks ? 2 : 1) + L::kNCh));
          ptx::tma_load_4d(sa, &tmDy, &full_bar[st], m0, -1, h0, img0);
          if (two_chunks) ptx::tma_load_4d(sa + kChunkA2, &tmDy, &full_bar[st], m0 + 64, -1, h0, img0);
#pragma unroll
          for (int c = 0; c < L::kNCh; ++c)
            ptx::tma_load_4d(sb + c * kChunkB2 + kPad2, &tmX, &full_bar[st], n0 + c * 64, -1, h0 + r - 1, img0);
        }
        __syncwarp();
      }
    } else if (warp >= 4) {
      const int cw = (warp - 4) >> 2;                            // consumer warpgroup = 64-channel chunk of dY
      const int et = threadIdx.x - 128;
      const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);
      const int cq = (lane & 3) * 2;
      constexpr int kVec = BLOCK_N / 4;
      float acc[3][BLOCK_N / 2];
      using Mma = ptx::WgmmaBf16<BLOCK_N, 1, 1>;
      const int ksteps = p.KB / kMmaK;
      for (int i = 0; i < num_kb; ++i) {
        const int st = i % kStages2;
        ptx::mbar_wait(&full_bar[st], (i / kStages2) & 1);
        const uint32_t sa = ptx::smem_u32(smem + st * L::kStage) + cw * kChunkA2;
        const uint32_t sb = ptx::smem_u32(smem + st * L::kStage) + 2 * kChunkA2 + kPad2;
        ptx::wgmma_fence();
        for (int k = 0; k < ksteps; ++k) {
          const uint64_t da = ptx::make_smem_desc(sa + k * 2048, kChunkA2, 1024);
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            const uint32_t start = sb + k * 2048 + (s - 1) * 128;
            const uint64_t db = ptx::make_smem_desc_bo(start, kChunkB2, 1024,
                                                       p.base_offset_mode ? ((start >> 7) & 7u) : 0u);
            Mma::mma(acc[s], da, db, (i | k) != 0 ? 1u : 0u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[st]);
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      uint8_t* sf = smem;
      int rows_valid = p.Cout - m0;
      if (rows_valid > kBlockM) rows_valid = kBlockM;
      const int64_t ldw = (int64_t)9 * p.Cin;
      const bool direct = gridDim.z == 1;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(sf + row * L::kPitch + (j * 8 + cq) * 4) = make_float2(acc[s][4 * j], acc[s][4 * j + 1]);
          *reinterpret_cast<float2*>(sf + (row + 8) * L::kPitch + (j * 8 + cq) * 4) = make_float2(acc[s][4 * j + 2], acc[s][4 * j + 3]);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int64_t col0 = (int64_t)(r * 3 + s) * p.Cin + n0;
#pragma unroll 1   // unrolled, this loop costs registers: the 128-column kernel spills more
        for (int f = et; f < rows_valid * kVec; f += kEpiThreads) {
          const int rr = f / kVec, c4 = (f % kVec) * 4;
          const float4 t = *reinterpret_cast<const float4*>(sf + rr * L::kPitch + c4 * 4);
          if (direct) {
            store_bf16x4(p.out + (int64_t)(m0 + rr) * ldw + col0 + c4, t, p.accumulate);
          } else {
            *reinterpret_cast<float4*>(p.part + ((int64_t)blockIdx.z * gridDim.x + blockIdx.x) * (kBlockM * 3 * BLOCK_N) +
                                       rr * (3 * BLOCK_N) + s * BLOCK_N + c4) = t;
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
    }
  }
}

struct Wgrad2Geometry {
  int WB = 0, BH = 0, NB = 0, KB = 0;
  bool ok = false;
};

// Box {Wb >= W + 1 columns starting at w = -1, BH rows, NB images}: Wb * BH * NB a multiple of 16 and <= kMaxKB2;
// fewest wasted (zero) K rows first, then the largest block.
Wgrad2Geometry plan_wgrad2(int N, int H, int W) {
  Wgrad2Geometry best;
  double best_eff = 0.0;
  if (W < 1 || H < 1 || N < 1) return best;
  for (int wb = W + 1; wb <= kMaxKB2 && wb <= W + 16; ++wb) {
    for (int nb = 1; nb <= 16 && nb <= N; nb *= 2) {
      for (int bh = 1; bh <= H; ++bh) {
        const int kb = wb * bh * nb;
        if (kb > kMaxKB2) break;
        if (kb % kMmaK != 0) continue;
        const int hb = (H + bh - 1) / bh, ng = (N + nb - 1) / nb;
        const double eff = (double)H * N * W / ((double)hb * bh * ng * nb * wb);
        if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && kb > best.KB)) {
          best_eff = eff;
          best.WB = wb; best.BH = bh; best.NB = nb; best.KB = kb; best.ok = true;
        }
      }
    }
  }
  return best;
}

int g_wgrad3_version = [] {
  const char* e = getenv("EDL_WGRAD3_V");
  return (e != nullptr && e[0] == '1') ? 1 : 2;
}();
int g_wgrad3_bo = [] {
  const char* e = getenv("EDL_WGRAD3_BO");
  return (e != nullptr && e[0] == '1') ? 1 : 0;
}();

// a split reduction needs a partial tile per (split, CTA); one that does not fit is an error, never a different path
const char* check_partials(const Conv3x3WgradArgs& a, int split, int64_t elems_per_split) {
  if (split > 1 && (a.partials == nullptr || a.partials_elems < split * elems_per_split))
    return "conv3x3_wgrad: split_k > 1 needs a partial-tile buffer of split * conv3x3_wgrad_tiles * 128 * 192 floats";
  return nullptr;
}

template <int BLOCK_N>
const char* launch_wgrad2(const Conv3x3WgradArgs& a, const Wgrad2Geometry& geo, cudaStream_t stream) {
  using L = W2Smem<BLOCK_N>;
  alignas(64) CUtensorMap tmDy, tmX;
  {
    const uint64_t dims[4] = {(uint64_t)a.Cout, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)a.Cout * 2, (uint64_t)a.W * a.Cout * 2, (uint64_t)a.H * a.W * a.Cout * 2};
    const uint32_t box[4] = {64, (uint32_t)geo.WB, (uint32_t)geo.BH, (uint32_t)geo.NB};
    if (const char* e = encode_tmap_bf16(&tmDy, a.dY, 4, dims, st, box)) return e;
  }
  {
    const uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)a.Cin * 2, (uint64_t)a.W * a.Cin * 2, (uint64_t)a.H * a.W * a.Cin * 2};
    const uint32_t box[4] = {64, (uint32_t)geo.WB, (uint32_t)geo.BH, (uint32_t)geo.NB};
    if (const char* e = encode_tmap_bf16(&tmX, a.X, 4, dims, st, box)) return e;
  }
  auto kern = conv3x3_wgrad2_kernel<BLOCK_N>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  Wgrad2Params p;
  p.Cout = a.Cout; p.Cin = a.Cin;
  p.BH = geo.BH; p.NB = geo.NB; p.KB = geo.KB;
  p.HB = (a.H + geo.BH - 1) / geo.BH;
  p.total_kb = p.HB * ((a.N + geo.NB - 1) / geo.NB);
  int split = a.split_k < 1 ? 1 : a.split_k;
  if (split > p.total_kb) split = p.total_kb;
  p.kb_per_split = (p.total_kb + split - 1) / split;
  split = (p.total_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.tiles_n = a.Cin / BLOCK_N;
  p.base_offset_mode = g_wgrad3_bo;
  const int tiles_m = (a.Cout + kBlockM - 1) / kBlockM;
  p.out = reinterpret_cast<__nv_bfloat16*>(a.dW);
  p.accumulate = a.accumulate ? 1 : 0;
  dim3 grid(tiles_m * p.tiles_n * 3, 1, split);
  if (const char* e = check_partials(a, split, (int64_t)grid.x * kBlockM * 3 * BLOCK_N)) return e;
  p.part = a.partials;
  kern<<<grid, kThreads, L::kTotal, stream>>>(tmDy, tmX, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cudaGetErrorString(e);
  if (split > 1) {
    splitk_reduce(a.partials, split, (int)grid.x, p.tiles_n, kBlockM, 3 * BLOCK_N, 3, a.Cin, a.Cout, 9 * a.Cin, a.dW,
                  (int64_t)9 * a.Cin, a.accumulate, stream);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

struct WgradGeometry {
  int BH = 0, NB = 0, KB = 0;
  bool ok = false;
};

// Pick the pixel box {W, BH rows, NB images}: W*BH*NB a multiple of 16 (MMA_K) and <= kMaxKB, as few
// zero-filled (out-of-image) rows as possible, then as many pixels per block as possible.
WgradGeometry plan_wgrad(int N, int H, int W) {
  WgradGeometry best;
  double best_eff = 0.0;
  if (W < 1 || W > kMaxKB || H < 1 || N < 1) return best;
  for (int nb = 1; nb <= 16 && nb <= N; nb *= 2) {
    for (int bh = 1; bh <= H; ++bh) {      // boxes never exceed the tensor extent (partial last blocks are zero-filled)
      const int kb = W * bh * nb;
      if (kb > kMaxKB) break;
      if (kb % kMmaK != 0) continue;
      const int hb = (H + bh - 1) / bh, ng = (N + nb - 1) / nb;
      const double eff = (double)H * N / ((double)hb * bh * ng * nb);
      if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && kb > best.KB)) {
        best_eff = eff;
        best.BH = bh; best.NB = nb; best.KB = kb; best.ok = true;
      }
    }
  }
  return best;
}

// version 1: TAPS filter taps per CTA (3: one row of the 3x3 convolution, 1: the 1x1 / stride-2 centre tap)
template <int TAPS>
const char* launch_wgrad1(const Conv3x3WgradArgs& a, cudaStream_t stream) {
  constexpr int kRows = TAPS == 3 ? 3 : 1;
  const bool s2 = a.stride == 2;
  const WgradGeometry geo = plan_wgrad(a.N, a.H, a.W);
  alignas(64) CUtensorMap tmDy, tmX;
  {
    const uint64_t dims[4] = {(uint64_t)a.Cout, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)a.Cout * 2, (uint64_t)a.W * a.Cout * 2, (uint64_t)a.H * a.W * a.Cout * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)geo.BH, (uint32_t)geo.NB};
    if (const char* e = encode_tmap_bf16(&tmDy, a.dY, 4, dims, st, box)) return e;
  }
  if (!s2) {
    const uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)a.Cin * 2, (uint64_t)a.W * a.Cin * 2, (uint64_t)a.H * a.W * a.Cin * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)geo.BH, (uint32_t)geo.NB};
    if (const char* e = encode_tmap_bf16(&tmX, a.X, 4, dims, st, box)) return e;
  } else {
    // the input is [N, 2H, 2W, Cin]: a box spanning 2W x 2BH elements with traversal stride 2 delivers the W x BH
    // input pixels that tap (r, s) pairs with the dY box -- same K-row order, no im2col, no subsample pass
    const uint64_t H2 = 2ull * a.H, W2 = 2ull * a.W;
    const uint64_t dims[4] = {(uint64_t)a.Cin, W2, H2, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)a.Cin * 2, W2 * a.Cin * 2, H2 * W2 * a.Cin * 2};
    const uint32_t box[4] = {64, (uint32_t)(2 * a.W), (uint32_t)(2 * geo.BH), (uint32_t)geo.NB};
    const uint32_t es[4] = {1, 2, 2, 1};
    if (const char* e = encode_tmap_strided(&tmX, a.X, 4, dims, st, box, es, 2)) return e;
  }
  auto kern = conv3x3_wgrad_kernel<TAPS>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  WgradParams p;
  p.Cout = a.Cout; p.Cin = a.Cin;
  p.BH = geo.BH; p.NB = geo.NB; p.KB = geo.KB;
  p.HB = (a.H + geo.BH - 1) / geo.BH;
  p.total_kb = p.HB * ((a.N + geo.NB - 1) / geo.NB);
  int split = a.split_k < 1 ? 1 : a.split_k;
  if (split > p.total_kb) split = p.total_kb;
  p.kb_per_split = (p.total_kb + split - 1) / split;
  split = (p.total_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.tiles_n = a.Cin / kBlockN;
  const int tiles_m = (a.Cout + kBlockM - 1) / kBlockM;
  p.out = reinterpret_cast<__nv_bfloat16*>(a.dW);
  p.accumulate = a.accumulate ? 1 : 0;
  p.stride = s2 ? 2 : 1;
  dim3 grid(tiles_m * p.tiles_n * kRows, 1, split);
  if (const char* e = check_partials(a, split, (int64_t)grid.x * kBlockM * TAPS * kBlockN)) return e;
  p.part = a.partials;
  kern<<<grid, kThreads, kSmemTotal, stream>>>(tmDy, tmX, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cudaGetErrorString(e);
  if (split > 1) {
    const int ld = TAPS * TAPS * a.Cin;
    splitk_reduce(a.partials, split, (int)grid.x, p.tiles_n, kBlockM, TAPS * kBlockN, TAPS, a.Cin, a.Cout, ld, a.dW,
                  (int64_t)ld, a.accumulate, stream);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

bool conv3x3_wgrad_supported(int N, int H, int W, int Cin, int Cout) {
  if (Cin % 64 != 0 || Cout % 64 != 0) return false;
  return g_wgrad3_version == 2 ? plan_wgrad2(N, H, W).ok : plan_wgrad(N, H, W).ok;
}

void set_wgrad3_version(int version, int base_offset_mode) {
  g_wgrad3_version = version == 1 ? 1 : 2;
  g_wgrad3_bo = base_offset_mode ? 1 : 0;
}
int get_wgrad3_version() { return g_wgrad3_version; }

bool conv3x3_wgrad_s2_supported(int N, int Ho, int Wo, int Cin, int Cout) {
  if (Cin % 64 != 0 || Cout % 64 != 0 || 2 * Wo > 256) return false;
  const WgradGeometry g = plan_wgrad(N, Ho, Wo);
  return g.ok && 2 * g.BH <= 256;
}

const char* conv3x3_wgrad_bf16(const Conv3x3WgradArgs& a, cudaStream_t stream) {
  const bool s2 = a.stride == 2;
  const bool k1 = a.ksize == 1;
  if (k1 && !s2) return "conv3x3_wgrad: the 1x1 weight gradient here is the stride-2 one";
  if (s2 ? !conv3x3_wgrad_s2_supported(a.N, a.H, a.W, a.Cin, a.Cout)
         : !conv3x3_wgrad_supported(a.N, a.H, a.W, a.Cin, a.Cout))
    return "conv3x3_wgrad: unsupported shape";
  if (a.dW == nullptr) return "conv3x3_wgrad: missing output";
  if (a.device >= 0) {
    cudaError_t e = cudaSetDevice(a.device);   // tensor-map encoding needs a bound context (see gemm.cu)
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  if (g_wgrad3_version == 2 && !s2) {
    const Wgrad2Geometry g2 = plan_wgrad2(a.N, a.H, a.W);
    return a.Cin % 128 == 0 ? launch_wgrad2<128>(a, g2, stream) : launch_wgrad2<64>(a, g2, stream);
  }
  return k1 ? launch_wgrad1<1>(a, stream) : launch_wgrad1<3>(a, stream);
}

// upper bound over both kernel versions, in CTAs of 64 Cin columns (sizes the partial-tile buffer)
int conv3x3_wgrad_tiles(int Cin, int Cout) { return ((Cout + kBlockM - 1) / kBlockM) * (Cin / kBlockN) * 3; }
// (tile, filter row) CTAs per split of the active version: what the split-K heuristic divides the SMs by
int conv3x3_wgrad_ctas(int Cin, int Cout) {
  const int bn = (g_wgrad3_version == 2 && Cin % 128 == 0) ? 128 : 64;
  return ((Cout + kBlockM - 1) / kBlockM) * (Cin / bn) * 3;
}

void conv3x3_wgrad_plan(int N, int H, int W, int* bh, int* nb, int* kb) {
  if (g_wgrad3_version == 2) {
    const Wgrad2Geometry g2 = plan_wgrad2(N, H, W);
    *bh = g2.ok ? g2.BH : 0;
    *nb = g2.ok ? g2.NB : 0;
    *kb = g2.ok ? g2.KB : 0;
    return;
  }
  const WgradGeometry g = plan_wgrad(N, H, W);
  *bh = g.ok ? g.BH : 0;
  *nb = g.ok ? g.NB : 0;
  *kb = g.ok ? g.KB : 0;
}

// stride-2 layers always run on the version-1 kernel: pixel blocks / CTAs per split for the split-K heuristic
int conv3x3_wgrad_s2_kblocks(int N, int Ho, int Wo) {
  const WgradGeometry g = plan_wgrad(N, Ho, Wo);
  if (!g.ok) return 0;
  return ((Ho + g.BH - 1) / g.BH) * ((N + g.NB - 1) / g.NB);
}

int conv3x3_wgrad_kblocks(int N, int H, int W) {
  if (g_wgrad3_version == 2) {
    const Wgrad2Geometry g2 = plan_wgrad2(N, H, W);
    if (!g2.ok) return 0;
    return ((H + g2.BH - 1) / g2.BH) * ((N + g2.NB - 1) / g2.NB);
  }
  const WgradGeometry g = plan_wgrad(N, H, W);
  if (!g.ok) return 0;
  return ((H + g.BH - 1) / g.BH) * ((N + g.NB - 1) / g.NB);
}

}  // namespace edl
