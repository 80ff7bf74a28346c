// 3x3 / stride-1 / pad-1 NHWC bf16 convolution as a wgmma implicit GEMM for sm_90a (SURVEY K1).
// The reference calls cuDNN through fluid.layers.conv2d (example/distill/resnet/models/resnet_vd.py:
// 153-162); this is an independent Hopper-native kernel.
//
// Implicit GEMM without an im2col buffer and without index math in the inner loop:
//
//   * the M tile is a PATCH of output pixels: BN images x BH rows x the full row width W
//     (BN*BH*W <= 128 accumulator rows), so one 4-D TMA box {64 channels, W, BH, BN} of the NHWC
//     input lands in shared memory exactly as a K-major [rows][64] wgmma operand tile;
//   * tap (r, s) of the filter is the SAME box shifted by (r-1, s-1) pixels -- rows / columns that
//     fall outside the image are zero-filled by the TMA unit, which IS the convolution padding;
//   * K loop = 9 taps x Cin/64 channel blocks, all accumulated into fp32 register tiles (64 rows per consumer
//     warpgroup); the weight tile of a tap is a plain 2-D box of the KRSC weight matrix
//     [Cout][9*Cin] (K-major for fprop, MN-major for dgrad -- no transposed weight copy);
//   * epilogue: accumulator registers -> bf16 -> swizzled staging -> one 4-D TMA store per 64 channels
//     (the store clips partial patches), with the train-mode BatchNorm statistics (per-channel sum and
//     sum of squares of the stored bf16 values) reduced from the staged tile.
//
// dgrad of a stride-1 3x3 conv is the same kernel on dY with mirrored shifts:
//   dX[n,h,w,ci] = sum_{r,s,co} dY[n, h+1-r, w+1-s, co] * W[co,r,s,ci].
//
// Warp roles as in gemm.cu: warp 0 TMA producer, warps 4..11 two consumer warpgroups (wgmma, then the epilogue).
#include <cuda.h>
#include <cstdio>

#include "gemm.h"
#include "kernels.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kMmaK = 16;
constexpr int kThreads = 384;   // producer warpgroup (one warp works) + two consumer warpgroups
constexpr int kEpiThreads = 256;

struct ConvParams {
  int n_img, H, W;
  int kc_blocks;     // input-channel blocks of 64 per tap
  int c_in_w;        // Cin of the weight tensor (column pitch of one tap in the [Cout][9*Cin] matrix)
  int n_out;         // output channels of this launch (fwd: Cout, dgrad: Cin)
  int BH, BN;        // patch rows / images per tile
  int tiles_h;       // ceil(H / BH)
  int dgrad;
  float* col_stats;
};

template <int BLOCK_N, int STAGES>
struct Smem {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kDBytes = kBlockM * BLOCK_N * 2;
  static constexpr int kTileBytes = STAGES * kStageBytes > kDBytes ? STAGES * kStageBytes : kDBytes;
  static constexpr int kBarOffset = kTileBytes;
  static constexpr int kTotal = kTileBytes + 256 + 1024;
};

EDL_DEVICE void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(ptx::smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <int BLOCK_N, int STAGES, bool DGRAD>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_wgmma_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                       const __grid_constant__ CUtensorMap tmY, const ConvParams p) {
  using L = Smem<BLOCK_N, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_n = (p.n_out + BLOCK_N - 1) / BLOCK_N;
  const int tile_m = blockIdx.x / tiles_n;
  const int n0 = (blockIdx.x % tiles_n) * BLOCK_N;
  const int img0 = (tile_m / p.tiles_h) * p.BN;
  const int h0 = (tile_m % p.tiles_h) * p.BH;
  const int rows_tile = p.BN * p.BH * p.W;          // accumulator rows that carry pixels
  const int num_kb = 9 * p.kc_blocks;
  const uint32_t a_bytes = (uint32_t)rows_tile * 128u;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmX);
    ptx::prefetch_tmap(&tmW);
    ptx::prefetch_tmap(&tmY);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ---------------------------------------------------------------- TMA producer
    if (lane == 0) {
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        const int tap = i / p.kc_blocks;
        const int kc = i - tap * p.kc_blocks;
        const int r = tap / 3, sft = tap - r * 3;
        const int dh = DGRAD ? 1 - r : r - 1;
        const int dw = DGRAD ? 1 - sft : sft - 1;
        ptx::mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * L::kStageBytes;
        uint8_t* sb = sa + L::kABytes;
        ptx::mbar_arrive_expect_tx(&full_bar[s], a_bytes + L::kBBytes);
        // activation patch shifted by the tap: out-of-image pixels arrive as zeros (= padding)
        ptx::tma_load_4d(sa, &tmX, &full_bar[s], kc * kBlockK, dw, h0 + dh, img0);
        if (!DGRAD) {
          // W as [Cout rows][9*Cin]: K-major tile, K offset = tap*Cin + kc*64
          ptx::tma_load_2d(sb, &tmW, &full_bar[s], tap * p.c_in_w + kc * kBlockK, n0);
        } else {
          // same matrix read MN-major: rows = co block (K), columns = ci (N) inside this tap
#pragma unroll
          for (int hh = 0; hh < BLOCK_N / 64; ++hh)
            ptx::tma_load_2d(sb + hh * 8192, &tmW, &full_bar[s], tap * p.c_in_w + n0 + hh * 64, kc * kBlockK);
        }
      }
    }
  } else if (warp >= 4) {
    // ---------------------------------------------------------------- consumers: MMA, then epilogue (warps 4..11)
    const int cw = (warp - 4) >> 2;                            // consumer warpgroup = 64-row half of the tile
    const int et = threadIdx.x - 128;
    const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // first accumulator row of this thread (second: + 8)
    const int cq = (lane & 3) * 2;
    float acc[BLOCK_N / 2];
    using Mma = ptx::WgmmaBf16<BLOCK_N, 0, DGRAD ? 1 : 0>;
    for (int i = 0; i < num_kb; ++i) {
      const int s = i % STAGES;
      ptx::mbar_wait(&full_bar[s], (i / STAGES) & 1);
      const uint32_t sa = ptx::smem_u32(smem + s * L::kStageBytes) + cw * 8192;
      const uint32_t sb = ptx::smem_u32(smem + s * L::kStageBytes) + L::kABytes;
      const uint64_t da0 = ptx::make_smem_desc(sa, 16, 1024);
      const uint64_t db0 = DGRAD ? ptx::make_smem_desc(sb, 8192, 1024) : ptx::make_smem_desc(sb, 16, 1024);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kMmaK; ++k)
        Mma::mma(acc, da0 + (uint64_t)(k * 2), db0 + (uint64_t)(k * (DGRAD ? 128 : 2)), (i | k) != 0 ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();
      if (i > 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[(i - 1) % STAGES]);
    }
    ptx::wgmma_wait<0>();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    uint8_t* sd = smem;  // the operand ring is drained: reuse it as the store staging tile
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      uint8_t* hp = sd + (j >> 3) * (kBlockM * 128) + cq * 2;
      *reinterpret_cast<__nv_bfloat162*>(hp + row * 128 + (((j & 7) ^ (row & 7)) << 4)) =
          __floats2bfloat162_rn(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<__nv_bfloat162*>(hp + (row + 8) * 128 + (((j & 7) ^ ((row + 8) & 7)) << 4)) =
          __floats2bfloat162_rn(acc[4 * j + 2], acc[4 * j + 3]);
    }
    ptx::fence_proxy_async_smem();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (et == 0) {
#pragma unroll
      for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh)
        if (n0 + hh * 64 < p.n_out) tma_store_4d(&tmY, sd + hh * (kBlockM * 128), n0 + hh * 64, 0, h0, img0);
      ptx::tma_store_commit();
    }
    if (p.col_stats != nullptr) {
      // rows of the patch that lie inside the tensor (partial patches at the bottom / last images)
      const int rows_per_img = p.BH * p.W;
      for (int col = et; col < BLOCK_N; col += kEpiThreads) {
        const bool valid = n0 + col < p.n_out;     // no early exit: the whole warp shuffles below
        const int half = col >> 6, cc = col & 63, chunk = cc >> 3, within = cc & 7;
        const uint8_t* base = sd + half * (kBlockM * 128) + within * 2;
        float s = 0.f, sq = 0.f;
        for (int b = 0; b < p.BN; ++b) {
          if (img0 + b >= p.n_img || !valid) break;
          int hv = p.H - h0;
          if (hv > p.BH) hv = p.BH;
          const int r_begin = b * rows_per_img, r_end = r_begin + hv * p.W;
#pragma unroll 4
          for (int rr = r_begin; rr < r_end; ++rr) {
            const __nv_bfloat16 hvv = *reinterpret_cast<const __nv_bfloat16*>(
                base + rr * 128 + ((chunk ^ (rr & 7)) << 4));
            const float v = __bfloat162float(hvv);
            s += v;
            sq = fmaf(v, v, sq);
          }
        }
        // four neighbouring columns -> one vector reduction (lane 4i collects lanes 4i..4i+3)
        const float s1 = __shfl_down_sync(0xffffffffu, s, 1), s2 = __shfl_down_sync(0xffffffffu, s, 2),
                    s3 = __shfl_down_sync(0xffffffffu, s, 3);
        const float q1 = __shfl_down_sync(0xffffffffu, sq, 1), q2 = __shfl_down_sync(0xffffffffu, sq, 2),
                    q3 = __shfl_down_sync(0xffffffffu, sq, 3);
        float* ps = &p.col_stats[n0 + col];
        float* pq = &p.col_stats[p.n_out + n0 + col];
        const int c4 = col & ~3;   // the decision is per group of four columns, identical in its 4 lanes
        const bool vec = (p.n_out % 4 == 0) && n0 + c4 + 3 < p.n_out &&
                         ((reinterpret_cast<uintptr_t>(&p.col_stats[n0 + c4]) & 15) == 0);
        if (vec) {
          if ((col & 3) == 0) {
            red_add_v4(ps, s, s1, s2, s3);
            red_add_v4(pq, sq, q1, q2, q3);
          }
        } else if (valid) {
          atomicAdd(ps, s);
          atomicAdd(pq, sq);
        }
      }
    }
    if (et == 0) ptx::tma_store_wait_read0();
  }
}

struct Geometry {
  int BH = 0, BN = 1, tiles_h = 0, tiles_img = 0;
  bool ok = false;
};

Geometry plan(int N, int H, int W) {
  Geometry g;
  if (W < 1 || W > kBlockM || H < 1) return g;
  int bh = kBlockM / W;
  if (bh > H) bh = H;
  // prefer a divisor of H (no partial patches) unless it wastes more than a quarter of the tile
  int best = bh;
  for (int d = bh; d >= 1; --d)
    if (H % d == 0) { best = d; break; }
  if (best * 4 < bh * 3) best = bh;
  g.BH = best;
  g.tiles_h = (H + g.BH - 1) / g.BH;
  g.BN = 1;
  if (g.BH == H) {
    int bn = kBlockM / (H * W);
    if (bn < 1) bn = 1;
    if (bn > N) bn = N;
    g.BN = bn;
  }
  g.tiles_img = (N + g.BN - 1) / g.BN;
  // TMA box dimensions are limited to 256 elements each
  g.ok = W <= 256 && g.BH <= 256 && g.BN <= 256;
  return g;
}

template <int BLOCK_N, int STAGES, bool DGRAD>
const char* launch(const Conv3x3Args& a, const Geometry& geo, cudaStream_t stream) {
  using L = Smem<BLOCK_N, STAGES>;
  const int cx = DGRAD ? a.Cout : a.Cin;   // channels of the tensor that is read
  const int cy = DGRAD ? a.Cin : a.Cout;   // channels of the tensor that is written
  alignas(64) CUtensorMap tmX, tmW, tmY;
  {
    const uint64_t dims[4] = {(uint64_t)cx, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cx * 2, (uint64_t)a.W * cx * 2, (uint64_t)a.H * a.W * cx * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)geo.BH, (uint32_t)geo.BN};
    if (const char* e = encode_tmap_bf16(&tmX, a.X, 4, dims, st, box)) return e;
  }
  {
    const uint64_t dims[4] = {(uint64_t)cy, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cy * 2, (uint64_t)a.W * cy * 2, (uint64_t)a.H * a.W * cy * 2};
    const uint32_t box[4] = {(uint32_t)(BLOCK_N < 64 ? BLOCK_N : 64), (uint32_t)a.W, (uint32_t)geo.BH,
                             (uint32_t)geo.BN};
    if (const char* e = encode_tmap_bf16(&tmY, a.Y, 4, dims, st, box)) return e;
  }
  {
    // KRSC weights as a matrix [Cout rows][9*Cin columns]
    const uint64_t dims[2] = {(uint64_t)9 * a.Cin, (uint64_t)a.Cout};
    const uint64_t st[1] = {(uint64_t)9 * a.Cin * 2};
    const uint32_t box[2] = {64, (uint32_t)(DGRAD ? kBlockK : BLOCK_N)};
    if (const char* e = encode_tmap_bf16(&tmW, a.Wt, 2, dims, st, box)) return e;
  }
  auto kern = conv3x3_wgmma_kernel<BLOCK_N, STAGES, DGRAD>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  ConvParams p;
  p.n_img = a.N; p.H = a.H; p.W = a.W;
  p.kc_blocks = cx / kBlockK;
  p.c_in_w = a.Cin;
  p.n_out = cy;
  p.BH = geo.BH; p.BN = geo.BN; p.tiles_h = geo.tiles_h;
  p.dgrad = DGRAD ? 1 : 0;
  p.col_stats = DGRAD ? nullptr : a.col_stats;
  const int tiles_n = (cy + BLOCK_N - 1) / BLOCK_N;
  dim3 grid(geo.tiles_img * geo.tiles_h * tiles_n, 1, 1);
  kern<<<grid, kThreads, L::kTotal, stream>>>(tmX, tmW, tmY, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

bool conv3x3_supported(int N, int H, int W, int Cin, int Cout, bool dgrad, int groups) {
  if (groups > 1) {
    // grouped fprop (persistent kernel): every N tile must lie inside one group
    if (dgrad || Cin % groups != 0 || Cout % groups != 0 || !persistent_gemm_enabled()) return false;
    const int cin_g = Cin / groups, cout_g = Cout / groups;
    if (cin_g % 64 != 0 || !(cout_g == 64 || cout_g % 128 == 0)) return false;
    return N >= 1 && plan(N, H, W).ok;
  }
  const int cx = dgrad ? Cout : Cin, cy = dgrad ? Cin : Cout;
  if (N < 1 || cx % 64 != 0 || cy % 8 != 0) return false;
  // dgrad reads the weight tile MN-major inside one tap: the N tile must not run into the next tap
  if (dgrad && cy % 64 != 0) return false;
  if (dgrad && cy > 64 && cy % 128 != 0) return false;
  return plan(N, H, W).ok;
}

const char* conv3x3_bf16(const Conv3x3Args& a, cudaStream_t stream) {
  if (!conv3x3_supported(a.N, a.H, a.W, a.Cin, a.Cout, a.dgrad, a.groups)) return "conv3x3: unsupported shape";
  if (!persistent_gemm_enabled() && (a.groups > 1 || a.col_scale != nullptr || a.col_shift != nullptr || a.relu))
    return "conv3x3: groups / inference epilogue need the persistent kernel";
  if (a.ksize != 3) return "conv3x3: a 1x1 / stride 2 convolution goes through conv1x1_s2_bf16";
  if (a.stride != 1 && (a.stride != 2 || a.dgrad || !persistent_gemm_enabled()))
    return "conv3x3: stride 2 is implemented for fprop on the persistent kernel only";
  if (a.device >= 0) {
    cudaError_t e = cudaSetDevice(a.device);   // tensor-map encoding needs a bound context (see gemm.cu)
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  const Geometry geo = plan(a.N, a.H, a.W);
  const int cy = a.dgrad ? a.Cin : a.Cout;
  if (persistent_gemm_enabled())
    return conv3x3_bf16_persistent(a, geo.BH, geo.BN, geo.tiles_h, geo.tiles_img, stream);
  if (!a.dgrad)
    return cy <= 64 ? launch<64, 4, false>(a, geo, stream) : launch<128, 3, false>(a, geo, stream);
  return cy <= 64 ? launch<64, 4, true>(a, geo, stream) : launch<128, 3, true>(a, geo, stream);
}

bool conv3x3_dgrad_s2_supported(int N, int Ho, int Wo, int Cin, int Cout) {
  return persistent_gemm_enabled() && conv3x3_supported(N, Ho, Wo, Cin, Cout, true, 1);
}

const char* conv3x3_dgrad_s2_bf16(const Conv3x3Args& a, cudaStream_t stream) {
  if (!conv3x3_dgrad_s2_supported(a.N, a.H, a.W, a.Cin, a.Cout)) return "conv3x3 stride-2 dgrad: unsupported shape";
  if (a.device >= 0) {
    cudaError_t e = cudaSetDevice(a.device);
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  const Geometry geo = plan(a.N, a.H, a.W);
  return conv3x3_dgrad_s2_persistent(a, geo.BH, geo.BN, geo.tiles_h, geo.tiles_img, stream);
}

bool conv1x1_s2_supported(int N, int Ho, int Wo, int Cin, int Cout, bool dgrad) {
  // the strided input map spans 2 Wo columns and 2 BH rows of the input: TMA boxes stop at 256 elements
  if (!persistent_gemm_enabled() || Wo < 1 || Ho < 1 || 2 * Wo > 256) return false;
  if (!conv3x3_supported(N, Ho, Wo, Cin, Cout, dgrad, 1)) return false;
  return 2 * plan(N, Ho, Wo).BH <= 256;
}

const char* conv1x1_s2_bf16(const Conv3x3Args& a, cudaStream_t stream) {
  if (a.ksize != 1 || a.stride != 2 || a.groups != 1) return "conv1x1_s2: ksize 1, stride 2, groups 1";
  if (!conv1x1_s2_supported(a.N, a.H, a.W, a.Cin, a.Cout, a.dgrad)) return "conv1x1_s2: unsupported shape";
  if (a.device >= 0) {
    cudaError_t e = cudaSetDevice(a.device);   // tensor-map encoding needs a bound context (see gemm.cu)
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  const Geometry geo = plan(a.N, a.H, a.W);
  if (a.dgrad) return conv1x1_dgrad_s2_persistent(a, geo.BH, geo.BN, geo.tiles_h, geo.tiles_img, stream);
  return conv3x3_bf16_persistent(a, geo.BH, geo.BN, geo.tiles_h, geo.tiles_img, stream);
}

}  // namespace edl
