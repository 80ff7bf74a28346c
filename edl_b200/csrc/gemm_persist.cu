// Persistent wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
// gemm.cu / conv3x3.cu launch one CTA per output tile.  The layers of ResNet50_vd at batch 32 have SHORT
// K loops (1..36 k-blocks), so a CTA's fixed work (barrier init, tensor-map fetch, pipeline fill, teardown)
// weighs on every tile.  This kernel keeps ONE CTA per SM alive and streams tiles through it:
//
//   warp 0      TMA producer: one smem ring shared by all tiles of the CTA, never drained between tiles
//               (the loads of tile i+1 are in flight while the consumers are in the epilogue of tile i)
//   warps 4..   consumer warpgroups (two, or four with 16 epilogue warps): each owns a 64-row half of the tile (and half
//               of its columns when there are four), issues its wgmma.mma_async into fp32 register accumulators, then runs
//               the epilogue: scale / shift / ReLU -> bf16 -> swizzled staging tile -> TMA store, BatchNorm statistics of
//               the stored values -> vector reductions
//
// Modes: 0 = D = A * B^T (B K-major: 1x1 conv fprop, FC), 1 = D = A * B (B MN-major: 1x1 conv dgrad),
//        2 = 3x3/s1/p1 conv fprop, 3 = 3x3/s1/p1 conv dgrad (see conv3x3.cu for the shifted-box trick).
#include <cuda.h>
#include <cstdio>
#include <cstdlib>

#include "gemm.h"
#include "kernels.h"
#include "launch.h"
#include "philox.cuh"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kMmaK = 16;
// BatchNorm statistics are accumulated per CTA in shared memory over ALL the tiles it processes and
// pushed to global memory once at the end: with one reduction request per tile and column group the
// requests queue in the L2 behind the few hot lines, which makes the 1568-tile 1x1 convs atomic-bound.
// N <= kMaxStatsN, else direct reductions.
constexpr int kMaxStatsN = 2048;

struct PersistParams {
  // GEMM view
  int M, N, K;
  int tiles_m, tiles_n;
  int num_kb;                 // k-blocks per tile (conv: 9 * kc_blocks)
  const float* col_scale;
  const float* col_shift;
  int relu;
  float* col_stats;
  const __nv_bfloat16* add_src;   // optional addend tile source (GEMM modes)
  long long ld_add;
  // fused BatchNorm-backward reduction (BNR kernels): D is the gradient dy of a BN layer's output
  const float* bn_mean;
  const float* bn_rstd;
  const float* bn_gamma;
  const float* bn_beta;
  float* bn_dsums;                // [2N]: += sum(dy_masked), sum(dy_masked * xhat)
  int bn_relu, bn_has_y;
  // ReLU mask bits of the BN output instead of y (1x1, N % 128 == 0): D is stored already masked
  int bn_has_mask;
  // conv view (modes 2, 3)
  int n_img, H, W, kc_blocks, c_in_w, BH, BN, tiles_h;
  int Wb;                         // halo layout: columns per image row of the A tile (W + 1)
  int b_res;                      // halo layout, one k-block per tap: the nine B tap tiles stay resident (see kRes)
  int cin_g, cout_g;              // grouped fprop: channels per group (cout_g == N for a dense conv)
  int stride;                     // conv fprop: 1, or 2 (input rows 2*h + r - 1; the columns come from the tensor map)
  // explicit tap list (conv modes; 0 = the nine standard taps): k-block i belongs to tap i / kc_blocks, which reads the
  // input box shifted by (tap_dh, tap_dw) and the weight tap tap_w.  Used by the stride-2 dgrad, which is four small
  // stride-1 convolutions over the output gradient -- one per parity class of the input pixel -- with 1, 2, 2 and 4 taps.
  int ntaps;
  signed char tap_dh[9], tap_dw[9], tap_w[9];
  // debug: per-phase clock64() stamps of CTA 0 (tools/trace_persist.py), [3 rows][kTraceTiles][8 phases]: row 0 producer, row 2 consumers
  long long* trace;
  // GELU == 2: the pre-activation u = acc * scale + shift, bf16 [M, N] with row pitch ld_aux
  __nv_bfloat16* aux;
  long long ld_aux;
  // GELU == 4: the dropout mask of the GEMM result
  PhiloxArgs drop;
};
constexpr int kTraceTiles = 16;
#define EDL_TRACE(role, tile, phase)                                                                    \
  do {                                                                                                  \
    if (p.trace != nullptr && blockIdx.x == 0 && (tile) < kTraceTiles)                                  \
      p.trace[((role) * kTraceTiles + (tile)) * 8 + (phase)] = clock64();                               \
  } while (0)

// ASTAGES > 0 selects the "haloed A tile" layout of the 3x3 convolution modes (see the kernel): the A tiles (one per filter
// ROW and k-block, 128 rows + a 1 KB zero pad on either side) and the B tiles (one per filter TAP) then live in two
// separate rings of ASTAGES and STAGES slots.
template <int BLOCK_N, int STAGES, int BNR = 0, int ASTAGES = 0>
struct PSmem {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kPad = 1024;
  static constexpr int kARegion = kABytes + 2 * kPad;              // halo layout: pad | tile | pad
  static constexpr int kARingBytes = ASTAGES * kARegion;
  static constexpr int kDBytes = kBlockM * BLOCK_N * 2;
  static constexpr int kRingBytes = ASTAGES > 0 ? kARingBytes + STAGES * kBBytes : STAGES * kStageBytes;
  static constexpr int kStatsBytes = 2 * kMaxStatsN * 4;   // CTA-local per-channel (sum, sum^2) accumulators
  static constexpr int kXOffset = kRingBytes + kDBytes;           // BNR: BN input tile x, then BN output tile y
  static constexpr int kXYBytes = BNR ? 2 * kDBytes : 0;
  static constexpr int kConstOffset = kXOffset + kXYBytes;        // BNR: mean, rstd, scale, shift of the tile's columns
  static constexpr int kConstBytes = BNR ? 4 * BLOCK_N * 4 : 0;    // float4 {mean, rstd, scale, shift} per column
  static constexpr int kStatsOffset = kConstOffset + kConstBytes;
  static constexpr int kBarOffset = kStatsOffset + kStatsBytes;
  static constexpr int kTotal = kBarOffset + 512 + 1024;
};

EDL_DEVICE void tma_store_4d_p(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(ptx::smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// BNR: TMA loads of the BN input (and output) tile of output tile (tm, nn0).  Called by a WHOLE warp (warp-uniform
// arguments); one elected lane issues.
template <int BLOCK_N, bool CONV>
EDL_DEVICE void issue_bn_tiles(const PersistParams& p, int tm, int nn0, int rows_tile, uint8_t* sx, uint8_t* sy,
                               const CUtensorMap* tmX, const CUtensorMap* tmY, uint64_t* bar) {
  const int mm0 = tm * kBlockM;
  const int im0 = CONV ? (tm / p.tiles_h) * p.BN : 0;
  const int hh0 = CONV ? (tm % p.tiles_h) * p.BH : 0;
  uint32_t halves = 0;
#pragma unroll
  for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh) halves += (nn0 + hh * 64 < p.N) ? 1u : 0u;
  const uint32_t tile_bytes = CONV ? (uint32_t)rows_tile * 128u : (uint32_t)(kBlockM * 128);
  if (ptx::elect_one()) {
    // the mask box is 16 bytes (128 columns) x 128 rows, unswizzled: row r at sy + 16 r
    const uint32_t mask_bytes = (!CONV && p.bn_has_mask) ? (uint32_t)(kBlockM * 16) : 0u;
    ptx::mbar_arrive_expect_tx(bar, halves * tile_bytes * (p.bn_has_y ? 2u : 1u) + mask_bytes);
    if (mask_bytes != 0) ptx::tma_load_2d(sy, tmY, bar, nn0 / 8, mm0);
#pragma unroll
    for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh) {
      if (nn0 + hh * 64 >= p.N) continue;
      if (!CONV) {
        ptx::tma_load_2d(sx + hh * (kBlockM * 128), tmX, bar, nn0 + hh * 64, mm0);
        if (p.bn_has_y) ptx::tma_load_2d(sy + hh * (kBlockM * 128), tmY, bar, nn0 + hh * 64, mm0);
      } else {
        ptx::tma_load_4d(sx + hh * (kBlockM * 128), tmX, bar, nn0 + hh * 64, 0, hh0, im0);
        if (p.bn_has_y) ptx::tma_load_4d(sy + hh * (kBlockM * 128), tmY, bar, nn0 + hh * 64, 0, hh0, im0);
      }
    }
  }
  __syncwarp();
}

// GELU: compile-time epilogue variants (0 = none; the other instantiations are unchanged by them).
//   1  inference: y = gelu(acc * scale + shift) with the erf form 0.5 v (1 + erf(v / sqrt 2)) in fp32 (the FFN1 GEMM of
//      a Transformer encoder, bias in col_shift)
//   2  training forward: the same y, and also u = acc * scale + shift as bf16 into p.aux (what the backward reads)
//   3  training dgrad (MODE 1): D = acc * gelu'(u) with gelu'(u) = Phi(u) + u phi(u) in fp32, u the bf16 addend tile
//      (FFN2's dgrad writes dU directly)
//   4  residual dropout (MODE 0): D = add + Z o (acc + shift), Z = keep * 1 / (1 - p) of the mask of p.drop at flat
//      index row * N + col (philox.cuh); dropout acts before the addend, and a dropped element stores the addend's bits.
//      The residual branches of a Transformer encoder layer (attention output projection, FFN2)
EDL_DEVICE float gelu_grad(float u) {
  return 0.5f * (1.f + erff(u * 0.70710678118654752f)) + u * 0.39894228040143268f * __expf(-0.5f * u * u);
}

template <int BLOCK_N, int STAGES, int MODE, int BNR, int ASTAGES, int EPIW, int GELU = 0>
__global__ void __launch_bounds__(128 + EPIW * 32, 1)
gemm_persist_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmAdd,
                    const __grid_constant__ CUtensorMap tmBnX, const __grid_constant__ CUtensorMap tmBnY,
                    const PersistParams p) {
  using L = PSmem<BLOCK_N, STAGES, BNR, ASTAGES>;
  constexpr int kEpiWarps = EPIW;
  constexpr int kThreads = 128 + kEpiWarps * 32;        // producer warpgroup (one warp works) + consumer warpgroups
  constexpr int kEpiThreads = kEpiWarps * 32;
  constexpr int kConsGroups = kEpiWarps / 4;             // consumer warpgroups: two row halves x kColGroups column groups
  constexpr int kColGroups = kEpiWarps / 8;
  static_assert(EPIW == 8 || EPIW == 16, "epilogue warps");
  static_assert(BLOCK_N / kColGroups >= 64 && (BLOCK_N / kColGroups) % 64 == 0, "a column group is whole 64-column halves");
  static_assert(BNR == 0 || BNR == 2, "BN-backward reduction: the column loop over the staged tiles");
  constexpr bool kConv = MODE >= 2;
  constexpr bool kBMN = MODE == 1 || MODE == 3;
  constexpr bool kDgrad = MODE == 3;
  // Haloed A tiles (3x3 / stride 1 convolutions): the pixel box of a tile is loaded with one extra column on the LEFT
  // (Wb = W + 1 columns starting at column -1, zero-filled by TMA), so tile row m = image_row * Wb + (w + 1) and the left /
  // right neighbour of a pixel is simply tile row m -/+ 1: the right neighbour of the last pixel of an image row is the
  // halo (zero) column of the next one.  The three taps of a filter row then read the SAME shared-memory tile through
  // wgmma descriptors whose start address is shifted by -128 / 0 / +128 bytes (the 128-byte swizzle is a function of the
  // shared-memory address, so whole-row shifts stay consistent with what TMA wrote; zero pads absorb the rows before
  // the first / after the last).  One A tile per filter row instead of one per tap: a third of the A traffic from L2.
  // The accumulator rows of the halo column are garbage and are dropped when the epilogue compacts the tile into the
  // dense [BN][BH][W] staging layout, so statistics, the fused BN-backward reduction and the TMA store are unchanged.
  constexpr bool kHalo = ASTAGES > 0;
  static_assert(!kHalo || kConv, "halo tiles: conv modes");
  // Resident B (64-channel layers / groups: one k-block per tap, the nine tap tiles of an N tile are 72 KB = the whole B
  // ring): the tiles are ordered N-major and every CTA takes a CONTIGUOUS run of them, so the weights of an N tile (a
  // group) are loaded once per run instead of once per tile -- slot j of the ring holds tap j, its full / empty barriers
  // flip once per N-tile change.  the grouped 14 x 14 layers of the teacher moved 229 MB
  // from L2 per launch, 147 MB of it the same 2.4 MB of weights fetched by each of the 64 pixel tiles.
  constexpr bool kRes = kHalo && BLOCK_N == 64 && STAGES == 9;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sd = smem + L::kRingBytes;                    // dedicated store-staging tile
  float* sstats = reinterpret_cast<float*>(smem + L::kStatsOffset);
  uint8_t* sx = smem + L::kXOffset;                       // BNR only
  uint8_t* sy = sx + L::kDBytes;
  float* sconst = reinterpret_cast<float*>(smem + L::kConstOffset);
  float* const stats_dst = BNR ? p.bn_dsums : p.col_stats;
  const bool local_stats = stats_dst != nullptr && p.N <= kMaxStatsN;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* add_bar = empty_bar + STAGES;                // addend tile landed in the staging buffer
  uint64_t* bn_bar = add_bar + 1;                        // BN x (/ y) tiles landed
  uint64_t* afull_bar = bn_bar + 1;                      // halo layout: the A ring's barriers
  uint64_t* aempty_bar = afull_bar + (kHalo ? ASTAGES : 0);
  static_assert((2 * STAGES + 2 + 2 * ASTAGES) * 8 <= 512, "barrier block");

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.tiles_m * p.tiles_n;
  const bool res = kRes && p.b_res != 0;
  int t_begin = blockIdx.x, t_end = total_tiles, t_step = gridDim.x;
  if (res) {
    // balanced contiguous runs: every CTA gets floor or ceil(total / grid) tiles (all SMs keep loads in flight)
    t_begin = (int)((long long)blockIdx.x * total_tiles / (int)gridDim.x);
    t_end = (int)((long long)(blockIdx.x + 1) * total_tiles / (int)gridDim.x);
    t_step = 1;
  }
  // tile index -> (M tile, first column): M-major normally (neighbouring CTAs share the A tile in L2), N-major when
  // B is resident
  // Incremental form for the role loops (an integer division by a run-time value is a long chain of dependent instructions,
  // and the epilogue needs the coordinates of this tile and the next)
  struct TileIt { int tm, ni; };
  const int step_m = res ? 0 : t_step / p.tiles_n, step_n = res ? 0 : t_step - (t_step / p.tiles_n) * p.tiles_n;
  auto tile_init = [&](int t) -> TileIt {
    if (res) {
      const int nt = t / p.tiles_m;
      return TileIt{t - nt * p.tiles_m, nt};
    }
    const int tm = t / p.tiles_n;
    return TileIt{tm, t - tm * p.tiles_n};
  };
  auto tile_next = [&](TileIt c) -> TileIt {
    if (res) {
      if (++c.tm >= p.tiles_m) { c.tm = 0; ++c.ni; }
    } else {
      c.tm += step_m;
      c.ni += step_n;
      if (c.ni >= p.tiles_n) { c.ni -= p.tiles_n; ++c.tm; }
    }
    return c;
  };
  auto tile_coords = [&](int t, int& tm, int& n0) {
    if (res) {
      const int nt = t / p.tiles_m;
      tm = t - nt * p.tiles_m;
      n0 = nt * BLOCK_N;
    } else {
      tm = t / p.tiles_n;
      n0 = (t - tm * p.tiles_n) * BLOCK_N;
    }
  };
  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    ptx::prefetch_tmap(&tmD);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kConsGroups);   // one arrival per consumer warpgroup
    }
    ptx::mbar_init(add_bar, 1);
    ptx::mbar_init(bn_bar, 1);
    for (int s = 0; s < ASTAGES; ++s) {
      ptx::mbar_init(&afull_bar[s], 1);
      ptx::mbar_init(&aempty_bar[s], kConsGroups);
    }
    ptx::fence_barrier_init();
  }
  if (local_stats)
    for (int i = threadIdx.x; i < 2 * p.N; i += kThreads) sstats[i] = 0.f;
  if (kHalo) {
    // pads AND tiles: TMA only ever writes the first rows_in rows of a tile, the rows behind them must read as zero
    for (int i = threadIdx.x; i < L::kARingBytes / 16; i += kThreads) ptx::sts128(ptx::smem_u32(smem) + i * 16, 0u, 0u, 0u, 0u);
    ptx::fence_proxy_async_smem();
  }
  __syncthreads();
  // everything above is CTA-local set-up; under programmatic dependent launch it overlapped the tail of the
  // previous kernel in the stream.  From here on global memory is touched.
  pdl_wait();
  pdl_launch_dependents();
  const int rows_tile = kConv ? p.BN * p.BH * p.W : kBlockM;            // rows of the (dense) output tile
  const int rows_in = kHalo ? p.BN * p.BH * p.Wb : rows_tile;          // rows of the A tile
  const uint32_t a_bytes = kConv ? (uint32_t)rows_in * 128u : (uint32_t)L::kABytes;

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    // The WHOLE warp runs the loops and waits on the barriers; one elected lane issues the copies.  With the loops
    // inside `if (lane == 0)` every tensor-map / barrier / coordinate operand is a per-thread value that the compiler has to
    // move into uniform registers with a vote + broadcast + retry sequence per operand.
    {
      uint32_t it = 0;
      [[maybe_unused]] uint32_t ita = 0;
      [[maybe_unused]] int cur_n0 = -1;
      [[maybe_unused]] uint32_t gcount = 0;
      TileIt cur = tile_init(t_begin);
      for (int t = t_begin; t < t_end; t += t_step, cur = tile_next(cur)) {
        const int tile_m = cur.tm, n0 = cur.ni * BLOCK_N;
        const int m0 = tile_m * kBlockM;
        const int img0 = kConv ? (tile_m / p.tiles_h) * p.BN : 0;
        const int h0 = kConv ? (tile_m % p.tiles_h) * p.BH : 0;
        if constexpr (kHalo) {
          // num_kb counts A steps here: (filter row r, k-block kc); each is followed by its three B tap tiles
          const int cbase_in = (MODE == 2) ? (n0 / p.cout_g) * p.cin_g : 0;
          const bool newg = n0 != cur_n0;
          if (newg) { cur_n0 = n0; ++gcount; }
          for (int i = 0; i < p.num_kb; ++i, ++ita) {
            const int r = i / p.kc_blocks, kc = i - r * p.kc_blocks;
            const int sa_i = ita % ASTAGES;
            ptx::mbar_wait(&aempty_bar[sa_i], ((ita / ASTAGES) & 1) ^ 1);
            if (ptx::elect_one()) {
              ptx::mbar_arrive_expect_tx(&afull_bar[sa_i], a_bytes);
              ptx::tma_load_4d(smem + sa_i * L::kARegion + L::kPad, &tmA, &afull_bar[sa_i], cbase_in + kc * kBlockK, -1,
                               h0 + (kDgrad ? 1 - r : r - 1), img0);
            }
            __syncwarp();
            if (res && !newg) continue;            // the taps of this N tile are already in their slots
            for (int sft = 0; sft < 3; ++sft, ++it) {
              const int s = res ? r * 3 + sft : (int)(it % STAGES);
              ptx::mbar_wait(&empty_bar[s], res ? ((gcount - 1) & 1) ^ 1 : ((it / STAGES) & 1) ^ 1);
              uint8_t* sb = smem + L::kARingBytes + s * L::kBBytes;
              const int tap = r * 3 + sft;
              if (ptx::elect_one()) {
                ptx::mbar_arrive_expect_tx(&full_bar[s], L::kBBytes);
                if (!kBMN) {
                  ptx::tma_load_2d(sb, &tmB, &full_bar[s], tap * p.c_in_w + kc * kBlockK, n0);
                } else {
#pragma unroll
                  for (int hh = 0; hh < BLOCK_N / 64; ++hh)
                    ptx::tma_load_2d(sb + hh * 8192, &tmB, &full_bar[s], tap * p.c_in_w + n0 + hh * 64, kc * kBlockK);
                }
              }
              __syncwarp();
            }
          }
        } else {
        for (int i = 0; i < p.num_kb; ++i, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          ptx::mbar_wait(&empty_bar[s], ph ^ 1);
          if (i == 0 && lane == 0) EDL_TRACE(0, (t - t_begin) / t_step, 0);
          uint8_t* sa = smem + s * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          if (!kConv) {
            const int k0 = i * kBlockK;
            if (ptx::elect_one()) {
              ptx::mbar_arrive_expect_tx(&full_bar[s], a_bytes + L::kBBytes);
              ptx::tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);
              if (!kBMN) {
                ptx::tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);
              } else {
#pragma unroll
                for (int hh = 0; hh < BLOCK_N / 64; ++hh)
                  ptx::tma_load_2d(sb + hh * 8192, &tmB, &full_bar[s], n0 + hh * 64, k0);
              }
            }
            __syncwarp();
          } else {
            int tap = i / p.kc_blocks;
            const int kc = i - tap * p.kc_blocks;
            int dh, dw;
            if (p.ntaps > 0) {
              dh = p.tap_dh[tap];
              dw = p.tap_dw[tap];
              tap = p.tap_w[tap];
            } else {
              const int r = tap / 3, sft = tap - r * 3;
              dh = kDgrad ? 1 - r : r - 1;
              dw = kDgrad ? 1 - sft : sft - 1;
            }
            // grouped fprop: the N tile lies in one group; its input channels start at group * cin_g
            const int cbase_in = (MODE == 2) ? (n0 / p.cout_g) * p.cin_g : 0;
            if (ptx::elect_one()) {
              ptx::mbar_arrive_expect_tx(&full_bar[s], a_bytes + L::kBBytes);
              ptx::tma_load_4d(sa, &tmA, &full_bar[s], cbase_in + kc * kBlockK, dw, h0 * p.stride + dh, img0);
              if (!kBMN) {
                ptx::tma_load_2d(sb, &tmB, &full_bar[s], tap * p.c_in_w + kc * kBlockK, n0);
              } else {
#pragma unroll
                for (int hh = 0; hh < BLOCK_N / 64; ++hh)
                  ptx::tma_load_2d(sb + hh * 8192, &tmB, &full_bar[s], tap * p.c_in_w + n0 + hh * 64, kc * kBlockK);
              }
            }
            __syncwarp();
          }
        }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers (warps 4..): MMA, then epilogue
    // Warpgroup cw owns the 64-row half (cw & 1) and the column group (cw >> 1) of every tile: it issues the
    // wgmma.mma_async of that part over the ring, then takes its fp32 register accumulators through the epilogue.
    const int ew = warp - 4;                 // 0..kEpiWarps-1
    const int q = warp & 3;                  // warp of the warpgroup: rows q * 16 .. q * 16 + 15 of its half
    const int cw = ew >> 2;
    const int grp = cw >> 1;                 // column group owned by this warpgroup
    const int et = threadIdx.x - 128;        // epilogue thread id
    constexpr int kColsPerGrp = BLOCK_N / kColGroups;
    const int row = (cw & 1) * 64 + q * 16 + (lane >> 2);   // first accumulator row of this thread (the second: + 8)
    const int cq = (lane & 3) * 2;                           // column of the thread inside an 8-column group
    const bool wg_lead = (threadIdx.x & 127) == 0;
    using Mma = ptx::WgmmaBf16<kColsPerGrp, 0, kBMN ? 1 : 0>;
    const uint32_t a_off = (uint32_t)(cw & 1) * 8192u;       // 64 rows of 128 bytes
    const uint32_t b_off = (uint32_t)grp * kColsPerGrp * 128u;
    int const_n0 = -1;
    uint32_t tc = 0, it = 0;
    [[maybe_unused]] uint32_t ita = 0;
    [[maybe_unused]] int cur_n0 = -1;
    [[maybe_unused]] uint32_t gcount = 0;
    // Column sums of the statistics / BN-backward loops stay in registers across the tiles of a run that share the N tile
    // (a thread always owns the same column pair) and go to the CTA-local accumulators once per run: fp32 atomicAdd on
    // shared memory is a compare-and-swap loop, and with kSplit threads per column hitting the same word four times per
    // tile it is a measurable part of a short-K tile.
    [[maybe_unused]] float run_s0 = 0.f, run_s1 = 0.f, run_q0 = 0.f, run_q1 = 0.f;
    TileIt cur = tile_init(t_begin);
    // halo layout: accumulator row -> row of the dense staging tile (fixed per thread; the halo column's rows are dropped)
    int srow[2] = {row, row + 8};
    bool store_ok[2] = {true, true};
    if (kHalo) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row + 8 * h;
        const int ir = r / p.Wb, cwd = r - ir * p.Wb;
        store_ok[h] = cwd != 0 && r < rows_in;
        srow[h] = ir * p.W + cwd - 1;
      }
    }
    for (int t = t_begin; t < t_end; t += t_step, ++tc) {
      const int tile_m = cur.tm, n0 = cur.ni * BLOCK_N;
      const bool has_next = t + t_step < t_end;
      [[maybe_unused]] const TileIt this_tile = cur;
      cur = tile_next(cur);
      const int next_tm = cur.tm, next_n0 = cur.ni * BLOCK_N;
      const int m0 = tile_m * kBlockM;
      const int img0 = kConv ? (tile_m / p.tiles_h) * p.BN : 0;
      const int h0 = kConv ? (tile_m % p.tiles_h) * p.BH : 0;
      if (et == 0) EDL_TRACE(2, tc, 0);
      // ---- main loop: this tile's k-blocks from the ring into the register accumulators
      float acc[kColsPerGrp / 2];
      if constexpr (kHalo) {
        bool newg = false, lastg = false;
        if (res) {
          newg = n0 != cur_n0;
          lastg = !has_next || next_n0 != n0;        // the slots are handed back after the last tile of the N tile
          if (newg) { cur_n0 = n0; ++gcount; }
        }
        for (int i = 0; i < p.num_kb; ++i, ++ita) {
          const int sa_i = ita % ASTAGES;
          ptx::mbar_wait(&afull_bar[sa_i], (ita / ASTAGES) & 1);
          const uint32_t sa = ptx::smem_u32(smem + sa_i * L::kARegion + L::kPad) + a_off;
          ptx::wgmma_fence();
          for (int sft = 0; sft < 3; ++sft) {
            const int s = res ? i * 3 + sft : (int)((it + sft) % STAGES);
            if (!res) ptx::mbar_wait(&full_bar[s], ((it + sft) / STAGES) & 1);
            else if (newg) ptx::mbar_wait(&full_bar[s], (gcount - 1) & 1);
            const uint32_t sb = ptx::smem_u32(smem + L::kARingBytes + s * L::kBBytes) + b_off;
            const int shift = (kDgrad ? 1 - sft : sft - 1) * 128;      // tile rows are 128 bytes
            const uint64_t da0 = ptx::make_smem_desc(sa + shift, 16, 1024);
            const uint64_t db0 = kBMN ? ptx::make_smem_desc(sb, 8192, 1024) : ptx::make_smem_desc(sb, 16, 1024);
#pragma unroll
            for (int k = 0; k < kBlockK / kMmaK; ++k)
              Mma::mma(acc, da0 + (uint64_t)(k * 2), db0 + (uint64_t)(k * (kBMN ? 128 : 2)), (i | sft | k) != 0 ? 1u : 0u);
          }
          ptx::wgmma_commit();
          ptx::wgmma_wait<0>();
          if (wg_lead) {
            for (int sft = 0; sft < 3; ++sft)
              if (!res || lastg) ptx::mbar_arrive(&empty_bar[res ? i * 3 + sft : (int)((it + sft) % STAGES)]);
            ptx::mbar_arrive(&aempty_bar[sa_i]);
          }
          it += 3;
        }
      } else {
        for (int i = 0; i < p.num_kb; ++i, ++it) {
          const int s = it % STAGES;
          ptx::mbar_wait(&full_bar[s], (it / STAGES) & 1);
          const uint32_t sa = ptx::smem_u32(smem + s * L::kStageBytes) + a_off;
          const uint32_t sb = ptx::smem_u32(smem + s * L::kStageBytes) + L::kABytes + b_off;
          const uint64_t da0 = ptx::make_smem_desc(sa, 16, 1024);
          const uint64_t db0 = kBMN ? ptx::make_smem_desc(sb, 8192, 1024) : ptx::make_smem_desc(sb, 16, 1024);
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / kMmaK; ++k)
            Mma::mma(acc, da0 + (uint64_t)(k * 2), db0 + (uint64_t)(k * (kBMN ? 128 : 2)), (i | k) != 0 ? 1u : 0u);
          ptx::wgmma_commit();
          // the MMAs of the previous k-block have read their stage: hand it back to the producer
          ptx::wgmma_wait<1>();
          if (i > 0 && wg_lead) ptx::mbar_arrive(&empty_bar[(it - 1) % STAGES]);
        }
        ptx::wgmma_wait<0>();
        if (wg_lead) ptx::mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      if (et == 0) EDL_TRACE(2, tc, 1);
      // the staging tile must have been read by the previous TMA store and by every stats thread
      // (bulk groups belong to the thread that issued the stores: always the elected lane of epilogue warp 0)
      if (ew == 0) {
        if (ptx::elect_one()) ptx::tma_store_wait_read0();
        __syncwarp();
      }
      asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory");
      // addend (if any): TMA-load its tile into the staging buffer (same swizzled layout as the output);
      // every thread then adds the pieces that belong to its accumulator registers
      const bool has_add = !kConv && p.add_src != nullptr;
      if (has_add) {
        if (ew == 0) {
          uint32_t halves = 0;
#pragma unroll
          for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh) halves += (n0 + hh * 64 < p.N) ? 1u : 0u;
          if (ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(add_bar, halves * (kBlockM * 128));
#pragma unroll
            for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh)
              if (n0 + hh * 64 < p.N) ptx::tma_load_2d(sd + hh * (kBlockM * 128), &tmAdd, add_bar, n0 + hh * 64, m0);
          }
          __syncwarp();
        }
        ptx::mbar_wait(add_bar, tc & 1);
      }
      if (BNR) {
        if (tc == 0 && ew == 0)                               // later tiles are prefetched one tile ahead
          issue_bn_tiles<BLOCK_N, kConv>(p, tile_m, n0, rows_tile, sx, sy, &tmBnX, &tmBnY, bn_bar);
        if (n0 != const_n0) {
          // per-column constants of the BN layer for this N tile (a CTA usually keeps its N tile)
          if (tc != 0) asm volatile("bar.sync 2, %0;" ::"n"(kEpiThreads) : "memory");   // everybody is done with the old ones
          if (et < BLOCK_N) {
            const int col = n0 + et;
            const bool in = col < p.N;
            const float mean = in ? p.bn_mean[col] : 0.f, rstd = in ? p.bn_rstd[col] : 0.f;
            const float scale = in ? p.bn_gamma[col] * rstd : 0.f;
            reinterpret_cast<float4*>(sconst)[et] = make_float4(mean, rstd, scale, in ? p.bn_beta[col] - mean * scale : 0.f);
          }
          asm volatile("bar.sync 2, %0;" ::"n"(kEpiThreads) : "memory");
          const_n0 = n0;
        }
      }
      if (et == 0) EDL_TRACE(2, tc, 2);
      // ---- accumulators -> addend / scale / shift / ReLU -> bf16 -> swizzled staging tile
      // BN ReLU mask bits (1x1 dgrad): the gradient is masked BEFORE it is staged, so what reaches HBM is dy * (y > 0)
      // and neither the reduction below nor the BN backward needs the mask again.  Bit b of byte j of a mask row is
      // column 8 j + b; this thread's columns are bytes grp * kColsPerGrp / 8 .. + kColsPerGrp / 8 - 1 of rows row, row + 8.
      // A mask word (four bytes) is loaded when the loop reaches its first column group.
      const bool bn_mask = BNR != 0 && !kConv && p.bn_has_mask != 0;
      [[maybe_unused]] uint32_t mword[2] = {0u, 0u};
      const uint32_t mbase = ptx::smem_u32(sy) + row * 16 + grp * (kColsPerGrp / 8);
      if (bn_mask) ptx::mbar_wait(bn_bar, tc & 1);
      // GELU == 4: keep bits of this thread's elements, bits 4 j + 2 h (+ 1) for column pair j of row row + 8 h, formed in
      // a rolled loop (unrolled into the epilogue, the Philox rounds would spill the accumulators)
      [[maybe_unused]] uint64_t kmask = 0;
      if constexpr (GELU == 4) {
        static_assert(kColsPerGrp / 8 * 4 <= 64, "keep bits of a thread");
        const PhiloxKey pk = philox_key(p.drop);
#pragma unroll 1
        for (int j = 0; j < kColsPerGrp / 8; ++j) {
          const uint64_t col = (uint64_t)(n0 + grp * kColsPerGrp + j * 8 + cq);
#pragma unroll
          for (int h = 0; h < 2; ++h)
            kmask |= (uint64_t)dropout_keep2(pk, (uint64_t)(m0 + row + 8 * h) * (uint64_t)p.N + col) << (4 * j + 2 * h);
        }
      }
#pragma unroll
      for (int j = 0; j < kColsPerGrp / 8; ++j) {
        const int tcol = grp * kColsPerGrp + j * 8 + cq;        // column inside the tile
        const int col = n0 + tcol;
        float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
        [[maybe_unused]] float addv[4];                         // GELU == 4: the addend, added after the dropout
        const uint32_t hp = ptx::smem_u32(sd) + (tcol >> 6) * (kBlockM * 128) + cq * 2;
        const int chunk = (tcol >> 3) & 7;
        if (has_add) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = row + 8 * h;
            const uint32_t w = ptx::lds32(hp + r * 128 + ((chunk ^ (r & 7)) << 4));
            const float2 t2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
            if constexpr (GELU == 3) {
              v[2 * h] *= gelu_grad(t2.x);
              v[2 * h + 1] *= gelu_grad(t2.y);
            } else if constexpr (GELU == 4) {
              addv[2 * h] = t2.x;
              addv[2 * h + 1] = t2.y;
            } else {
              v[2 * h] += t2.x;
              v[2 * h + 1] += t2.y;
            }
          }
        }
        if (bn_mask) {
          if ((j & 3) == 0) {
            mword[0] = ptx::lds32(mbase + (j >> 2) * 4);
            mword[1] = ptx::lds32(mbase + 8 * 16 + (j >> 2) * 4);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t bits = mword[h] >> ((j & 3) * 8 + cq);
            v[2 * h] = (bits & 1u) ? v[2 * h] : 0.f;
            v[2 * h + 1] = (bits & 2u) ? v[2 * h + 1] : 0.f;
          }
        }
        if (!BNR) {
          if (p.col_scale != nullptr) {
            const float s0 = col < p.N ? __ldg(p.col_scale + col) : 0.f, s1 = col + 1 < p.N ? __ldg(p.col_scale + col + 1) : 0.f;
            v[0] *= s0; v[1] *= s1; v[2] *= s0; v[3] *= s1;
          }
          if (p.col_shift != nullptr) {
            const float s0 = col < p.N ? __ldg(p.col_shift + col) : 0.f, s1 = col + 1 < p.N ? __ldg(p.col_shift + col + 1) : 0.f;
            v[0] += s0; v[1] += s1; v[2] += s0; v[3] += s1;
          }
          if (p.relu) {
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = fmaxf(v[e], 0.f);
          }
          if constexpr (GELU == 2) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = m0 + row + 8 * h;
              if (r < p.M && col < p.N)
                *reinterpret_cast<__nv_bfloat162*>(p.aux + (int64_t)r * p.ld_aux + col) =
                    __floats2bfloat162_rn(v[2 * h], v[2 * h + 1]);
            }
          }
          if constexpr (GELU == 1 || GELU == 2) {
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = 0.5f * v[e] * (1.f + erff(v[e] * 0.70710678118654752f));
          }
          if constexpr (GELU == 4) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t kb = (uint32_t)(kmask >> (4 * j + 2 * h));
              v[2 * h] = (kb & 1u) ? fmaf(v[2 * h], p.drop.scale, addv[2 * h]) : addv[2 * h];
              v[2 * h + 1] = (kb & 2u) ? fmaf(v[2 * h + 1], p.drop.scale, addv[2 * h + 1]) : addv[2 * h + 1];
            }
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const __nv_bfloat162 pk = __floats2bfloat162_rn(v[2 * h], v[2 * h + 1]);
          if (store_ok[h])
            asm volatile("st.shared.u32 [%0], %1;" ::"r"(hp + srow[h] * 128 + ((chunk ^ (srow[h] & 7)) << 4)),
                         "r"(*reinterpret_cast<const uint32_t*>(&pk))
                         : "memory");
        }
      }
      if (et == 0) EDL_TRACE(2, tc, 3);
      ptx::fence_proxy_async_smem();
      asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory");
      if (et == 0) EDL_TRACE(2, tc, 4);
      if (ew == 0) {
        if (ptx::elect_one()) {
#pragma unroll
          for (int hh = 0; hh < (BLOCK_N + 63) / 64; ++hh) {
            if (n0 + hh * 64 >= p.N) continue;
            if (!kConv) ptx::tma_store_2d(&tmD, sd + hh * (kBlockM * 128), n0 + hh * 64, m0);
            else tma_store_4d_p(&tmD, sd + hh * (kBlockM * 128), n0 + hh * 64, 0, h0, img0);
          }
          ptx::tma_store_commit();
        }
        __syncwarp();
      }
      if (BNR == 2) {
        // BatchNorm-backward reduction of the tile just staged: per channel sum(dy_m) and sum(dy_m * xhat), dy_m = the
        // STORED bf16 gradient masked by the layer's ReLU.  Same scheme as the forward statistics below -- a thread owns
        // a pair of adjacent columns and every kSplit-th row, eight independent row loads in flight -- reading the
        // gradient from the staging tile and x (/ y) from the tiles the producer fetched by TMA.
        ptx::mbar_wait(bn_bar, tc & 1);
        if (et == 0) EDL_TRACE(2, tc, 5);
        constexpr int kPairs = BLOCK_N / 2;
        constexpr int kSplit = kEpiThreads / kPairs;
        const int pair = et % kPairs;
        const int part = et / kPairs;
        const int col = pair * 2;
        const bool valid = n0 + col < p.N;
        const int half = col >> 6, cc = col & 63, chunk = cc >> 3, within = cc & 7;
        const uint32_t toff = half * (kBlockM * 128) + within * 2;
        const uint32_t based = ptx::smem_u32(sd) + toff, basex = ptx::smem_u32(sx) + toff, basey = ptx::smem_u32(sy) + toff;
        const float4 k0 = reinterpret_cast<const float4*>(sconst)[col];          // mean, rstd, scale, shift
        const float4 k1 = reinterpret_cast<const float4*>(sconst)[col + 1];
        // with mask bits the staged gradient is already masked
        const bool relu = p.bn_relu != 0 && !bn_mask, has_y = p.bn_has_y != 0;
        // s = sum(dy_m), q = sum(dy_m * x) over this thread's rows; sum(dy_m * xhat) = rstd * (q - mean * s) is formed once
        // per thread and tile below (two instructions per element less than normalising x in the loop).  With the BN
        // OUTPUT at hand the ReLU mask is a packed bf16 compare and a multiplication by 1.0 / 0.0 (exact).
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
        const __nv_bfloat162 zero2 = __floats2bfloat162_rn(0.f, 0.f);
        auto row_update = [&](uint32_t wd, uint32_t wx, uint32_t wy) {
          __nv_bfloat162 d2 = *reinterpret_cast<const __nv_bfloat162*>(&wd);
          const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wx));
          float2 d;
          if (relu && has_y) {
            d2 = __hmul2(d2, __hgt2(*reinterpret_cast<const __nv_bfloat162*>(&wy), zero2));
            d = __bfloat1622float2(d2);
          } else {
            d = __bfloat1622float2(d2);
            if (relu) {
              d.x = fmaf(x.x, k0.z, k0.w) > 0.f ? d.x : 0.f;
              d.y = fmaf(x.y, k1.z, k1.w) > 0.f ? d.y : 0.f;
            }
          }
          s0 += d.x; q0 = fmaf(d.x, x.x, q0);
          s1 += d.y; q1 = fmaf(d.y, x.y, q1);
        };
        // Row r of a staged tile sits at r * 128 + ((chunk ^ (r & 7)) << 4).  A thread visits rows r0, r0 + kSplit, ...:
        // with kSplit a multiple of 4 the swizzle term takes two values (even / odd steps), so two base addresses plus
        // compile-time offsets replace five address instructions per row and load.
        constexpr bool kFastRows = kSplit % 4 == 0;      // (the 256-column kernels carry no reduction; they only compile this)
        auto accum_rows = [&](int r_begin, int r_end) {
          int rr = r_begin + part;
          uint32_t o0 = rr * 128 + ((chunk ^ (rr & 7)) << 4), o1 = (rr + kSplit) * 128 + ((chunk ^ ((rr + kSplit) & 7)) << 4);
          for (; rr + 7 * kSplit < r_end; rr += 8 * kSplit, o0 += 8 * kSplit * 128, o1 += 8 * kSplit * 128) {
            uint32_t wd[8], wx[8], wy[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int r = rr + u * kSplit;
              const uint32_t o = kFastRows ? ((u & 1) ? o1 : o0) + (u >> 1) * (2 * kSplit * 128)
                                           : (uint32_t)(r * 128 + ((chunk ^ (r & 7)) << 4));
              wd[u] = ptx::lds32(based + o);
              wx[u] = ptx::lds32(basex + o);
              wy[u] = has_y ? ptx::lds32(basey + o) : 0u;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) row_update(wd[u], wx[u], wy[u]);
          }
#pragma unroll 1
          for (int u = 0; rr < r_end; rr += kSplit, ++u) {
            const uint32_t o = kFastRows ? ((u & 1) ? o1 : o0) + (u >> 1) * (2 * kSplit * 128)
                                         : (uint32_t)(rr * 128 + ((chunk ^ (rr & 7)) << 4));
            row_update(ptx::lds32(based + o), ptx::lds32(basex + o), has_y ? ptx::lds32(basey + o) : 0u);
          }
        };
        if (valid) {
          // only rows that are real pixels of the tensor: the others hold stale shared memory
          if (!kConv) {
            int rows_valid = p.M - m0;
            if (rows_valid > kBlockM) rows_valid = kBlockM;
            accum_rows(0, rows_valid);
          } else {
            const int rows_per_img = p.BH * p.W;
            int hv = p.H - h0;
            if (hv > p.BH) hv = p.BH;
            for (int b = 0; b < p.BN && img0 + b < p.n_img; ++b) accum_rows(b * rows_per_img, b * rows_per_img + hv * p.W);
          }
          run_s0 += s0; run_q0 += (q0 - k0.x * s0) * k0.y;          // k = {mean, rstd, scale, shift}
          run_s1 += s1; run_q1 += (q1 - k1.x * s1) * k1.y;
          if (!has_next || next_n0 != n0) {
            if (local_stats) {
              atomicAdd(&sstats[n0 + col], run_s0);
              atomicAdd(&sstats[p.N + n0 + col], run_q0);
              if (n0 + col + 1 < p.N) {
                atomicAdd(&sstats[n0 + col + 1], run_s1);
                atomicAdd(&sstats[p.N + n0 + col + 1], run_q1);
              }
            } else {
              atomicAdd(&p.bn_dsums[n0 + col], run_s0);
              atomicAdd(&p.bn_dsums[p.N + n0 + col], run_q0);
              if (n0 + col + 1 < p.N) {
                atomicAdd(&p.bn_dsums[n0 + col + 1], run_s1);
                atomicAdd(&p.bn_dsums[p.N + n0 + col + 1], run_q1);
              }
            }
          }
        }
        if (!has_next || next_n0 != n0) run_s0 = run_s1 = run_q0 = run_q1 = 0.f;
        // everybody is done with this tile's x / y: fetch the next tile's while its MMAs run
        if (et == 0) EDL_TRACE(2, tc, 6);
        asm volatile("bar.sync 3, %0;" ::"n"(kEpiThreads) : "memory");
        if (et == 0) EDL_TRACE(2, tc, 7);
        if (ew == 0 && has_next)
          issue_bn_tiles<BLOCK_N, kConv>(p, next_tm, next_n0, rows_tile, sx, sy, &tmBnX, &tmBnY, bn_bar);
      }
      if (!BNR && et == 0) EDL_TRACE(2, tc, 5);
      if (!BNR && p.col_stats != nullptr) {
        // Per-channel sum / sum of squares of the STORED bf16 values, from the staged tile.  A thread owns
        // a PAIR of adjacent columns (one 32-bit shared load per row) and every kSplit-th row; eight
        // independent loads are in flight per thread (a one-column, one-accumulator loop exposes the
        // shared-memory latency of every row).
        constexpr int kPairs = BLOCK_N / 2;                    // 64 (N=128) or 32 (N=64)
        constexpr int kSplit = kEpiThreads / kPairs;           // 4 or 8 row subsets
        const int pair = et % kPairs;
        const int part = et / kPairs;
        const int col = pair * 2;
        const bool valid = n0 + col < p.N;
        const int half = col >> 6, cc = col & 63, chunk = cc >> 3, within = cc & 7;
        const uint32_t base = ptx::smem_u32(sd) + half * (kBlockM * 128) + within * 2;
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
        constexpr bool kFastRows = kSplit % 4 == 0;
        auto accum_rows = [&](int r_begin, int r_end) {      // addressing: see the BN-backward loop above
          int rr = r_begin + part;
          uint32_t o0 = base + rr * 128 + ((chunk ^ (rr & 7)) << 4);
          uint32_t o1 = base + (rr + kSplit) * 128 + ((chunk ^ ((rr + kSplit) & 7)) << 4);
          for (; rr + 7 * kSplit < r_end; rr += 8 * kSplit, o0 += 8 * kSplit * 128, o1 += 8 * kSplit * 128) {
            uint32_t w[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int r = rr + u * kSplit;
              w[u] = ptx::lds32(kFastRows ? ((u & 1) ? o1 : o0) + (u >> 1) * (2 * kSplit * 128)
                                          : base + r * 128 + ((chunk ^ (r & 7)) << 4));
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[u]));
              s0 += v.x; q0 = fmaf(v.x, v.x, q0);
              s1 += v.y; q1 = fmaf(v.y, v.y, q1);
            }
          }
#pragma unroll 1
          for (int u = 0; rr < r_end; rr += kSplit, ++u) {
            const uint32_t w = ptx::lds32(kFastRows ? ((u & 1) ? o1 : o0) + (u >> 1) * (2 * kSplit * 128)
                                                    : base + rr * 128 + ((chunk ^ (rr & 7)) << 4));
            const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
            s0 += v.x; q0 = fmaf(v.x, v.x, q0);
            s1 += v.y; q1 = fmaf(v.y, v.y, q1);
          }
        };
        if (valid) {
          if (!kConv) {
            int rows_valid = p.M - m0;
            if (rows_valid > kBlockM) rows_valid = kBlockM;
            accum_rows(0, rows_valid);
          } else {
            const int rows_per_img = p.BH * p.W;
            int hv = p.H - h0;
            if (hv > p.BH) hv = p.BH;
            for (int b = 0; b < p.BN && img0 + b < p.n_img; ++b) accum_rows(b * rows_per_img, b * rows_per_img + hv * p.W);
          }
        }
        if (et == 0) EDL_TRACE(2, tc, 7);
        run_s0 += s0; run_s1 += s1; run_q0 += q0; run_q1 += q1;
        const bool run_end = !has_next || next_n0 != n0;
        if (run_end) { s0 = run_s0; s1 = run_s1; q0 = run_q0; q1 = run_q1; run_s0 = run_s1 = run_q0 = run_q1 = 0.f; }
        if (!run_end) {
          // the sums travel on in registers
        } else if (local_stats) {
          if (valid) {
            atomicAdd(&sstats[n0 + col], s0);
            atomicAdd(&sstats[p.N + n0 + col], q0);
            if (n0 + col + 1 < p.N) {
              atomicAdd(&sstats[n0 + col + 1], s1);
              atomicAdd(&sstats[p.N + n0 + col + 1], q1);
            }
          }
        } else {
          // lanes 2i, 2i+1 hold four neighbouring columns -> one vector reduction each for sum and sum^2
          const float s2 = __shfl_down_sync(0xffffffffu, s0, 1), s3 = __shfl_down_sync(0xffffffffu, s1, 1);
          const float q2 = __shfl_down_sync(0xffffffffu, q0, 1), q3 = __shfl_down_sync(0xffffffffu, q1, 1);
          const int c4 = col & ~3;
          float* ps4 = &p.col_stats[n0 + c4];
          const bool vec = (p.N % 4 == 0) && n0 + c4 + 3 < p.N && ((reinterpret_cast<uintptr_t>(ps4) & 15) == 0);
          if (vec) {
            if ((pair & 1) == 0) {
              red_add_v4(ps4, s0, s1, s2, s3);
              red_add_v4(ps4 + p.N, q0, q1, q2, q3);
            }
          } else if (valid) {
            atomicAdd(&p.col_stats[n0 + col], s0);
            atomicAdd(&p.col_stats[p.N + n0 + col], q0);
            if (n0 + col + 1 < p.N) {
              atomicAdd(&p.col_stats[n0 + col + 1], s1);
              atomicAdd(&p.col_stats[p.N + n0 + col + 1], q1);
            }
          }
        }
        if (et == 0) EDL_TRACE(2, tc, 6);
      }
    }
    if (local_stats) {
      // one flush per CTA: only the column groups this CTA touched are non-zero
      asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory");
      const bool vec_ok = (p.N % 4 == 0) && ((reinterpret_cast<uintptr_t>(stats_dst) & 15) == 0);
      if (vec_ok) {
        for (int i = et * 4; i < 2 * p.N; i += kEpiThreads * 4) {
          const float4 v = *reinterpret_cast<const float4*>(&sstats[i]);
          if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) red_add_v4(&stats_dst[i], v.x, v.y, v.z, v.w);
        }
      } else {
        for (int i = et; i < 2 * p.N; i += kEpiThreads)
          if (sstats[i] != 0.f) atomicAdd(&stats_dst[i], sstats[i]);
      }
    }
    if (ew == 0) {
      if (ptx::elect_one()) ptx::tma_store_wait_read0();
      __syncwarp();
    }
  }
}

bool g_persistent = true;
long long* g_trace = nullptr;
bool g_wide_tiles = [] {
  const char* e = getenv("EDL_GEMM_WIDE");
  return !(e != nullptr && e[0] == '0');
}();
// haloed A tiles for the 3x3 / stride 1 convolutions (EDL_CONV_HALO=0 keeps the one-box-per-tap version for A/B)
bool g_conv_halo = [] {
  const char* e = getenv("EDL_CONV_HALO");
  return !(e != nullptr && e[0] == '0');
}();

bool g_conv_bres = [] {
  const char* e = getenv("EDL_CONV_BRES");
  return !(e != nullptr && e[0] == '0');
}();

// tile geometry with Wb = W + 1 columns per image row (conv3x3.cu's planner with the row width replaced)
bool halo_geometry(int N, int H, int W, int* BH, int* BN, int* tiles_h, int* tiles_img) {
  const int wb = W + 1;
  if (W < 1 || wb > kBlockM || H < 1) return false;
  int bh = kBlockM / wb;
  if (bh > H) bh = H;
  int best = bh;
  for (int d = bh; d >= 1; --d)
    if (H % d == 0) { best = d; break; }
  if (best * 4 < bh * 3) best = bh;
  int bn = 1;
  if (best == H) {
    bn = kBlockM / (H * wb);
    if (bn < 1) bn = 1;
    if (bn > N) bn = N;
  }
  *BH = best; *BN = bn;
  *tiles_h = (H + best - 1) / best;
  *tiles_img = (N + bn - 1) / bn;
  return true;
}

// 16 consumer warps (four warpgroups, 64 rows x half of the columns each) are selectable (EDL_EPI_WARPS=16); the default is 8.
bool g_epi16 = [] {
  const char* e = getenv("EDL_EPI_WARPS");
  return e != nullptr && e[0] == '1' && e[1] == '6';
}();

template <int BLOCK_N, int STAGES, int MODE, int BNR, int ASTAGES, int EPIW, int GELU>
const char* launch_pe(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const PersistParams& p,
                     cudaStream_t stream, const CUtensorMap* tmAdd = nullptr, const CUtensorMap* tmBnX = nullptr,
                     const CUtensorMap* tmBnY = nullptr) {
  using L = PSmem<BLOCK_N, STAGES, BNR, ASTAGES>;
  static_assert(L::kTotal <= 227 * 1024, "shared memory budget");
  constexpr int kThreads = 128 + EPIW * 32;
  auto kern = gemm_persist_kernel<BLOCK_N, STAGES, MODE, BNR, ASTAGES, EPIW, GELU>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  const int total = p.tiles_m * p.tiles_n;
  const int grid = total < kNumSMs ? total : kNumSMs;
  PersistParams pt = p;
  pt.trace = g_trace;
  cudaError_t e = launch_pdl(kern, dim3(grid), dim3(kThreads), (size_t)L::kTotal, stream, tmA, tmB, tmD,
                             tmAdd != nullptr ? *tmAdd : tmD, tmBnX != nullptr ? *tmBnX : tmD,
                             tmBnY != nullptr ? *tmBnY : tmD, pt);
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

template <int BLOCK_N, int STAGES, int MODE, int BNR = 0, int ASTAGES = 0, int GELU = 0>
const char* launch_p(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const PersistParams& p,
                     cudaStream_t stream, const CUtensorMap* tmAdd = nullptr, const CUtensorMap* tmBnX = nullptr,
                     const CUtensorMap* tmBnY = nullptr) {
  if constexpr (BLOCK_N >= 128 && GELU != 4) {    // (the residual-dropout epilogue spills with 16 warps' registers)
    if (g_epi16)
      return launch_pe<BLOCK_N, STAGES, MODE, BNR, ASTAGES, 16, GELU>(tmA, tmB, tmD, p, stream, tmAdd, tmBnX, tmBnY);
  }
  return launch_pe<BLOCK_N, STAGES, MODE, BNR, ASTAGES, 8, GELU>(tmA, tmB, tmD, p, stream, tmAdd, tmBnX, tmBnY);
}

const char* tmap2d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_elems,
                   uint32_t box_inner, uint32_t box_outer) {
  const uint64_t dims[2] = {inner, outer};
  const uint64_t st[1] = {pitch_elems * 2};
  const uint32_t box[2] = {box_inner, box_outer};
  return encode_tmap_bf16(out, ptr, 2, dims, st, box);
}

}  // namespace

namespace {
void fill_bn(PersistParams& p, const BnBwdFuse& bn) {
  p.bn_mean = bn.mean; p.bn_rstd = bn.rstd; p.bn_gamma = bn.gamma; p.bn_beta = bn.beta;
  p.bn_dsums = bn.dsums;
  p.bn_relu = bn.relu ? 1 : 0;
  p.bn_has_y = (bn.relu && bn.y != nullptr) ? 1 : 0;
  p.bn_has_mask = (bn.relu && bn.mask != nullptr) ? 1 : 0;
}
}  // namespace

int get_bnr_mode() { return 2; }   // the column-pair loop over the staged tiles
void set_persistent_gemm(bool on) { g_persistent = on; }
void set_wide_gemm_tiles(bool on) { g_wide_tiles = on; }
bool persistent_gemm_enabled() { return g_persistent; }

// GEMM front end (EPI 0 semantics of gemm.cu; A K-major)
const char* gemm_bf16_persistent(const GemmArgs& g, cudaStream_t stream) {
  alignas(64) CUtensorMap tmA, tmB, tmD;
  const bool n64 = g.N <= 64;
  // 128 x 256 tiles for the compute-heavy GEMMs (the teacher's 1x1 convolutions: N = 512 .. 4096, K = 256 .. 4096):
  // a 128 x 128 tile needs 32 KB of operands per 256 tensor-core cycles = 128 B / clk / SM, about twice what the
  // L2 -> SM path delivers when every SM pulls; with N = 256 the
  // A tile is reused twice as often and the requirement drops to 96 B / clk.
  // (not with the GELU epilogue: with the erf expansion the 256-column tile spills its accumulators)
  const bool wide = g_wide_tiles && !g.gelu && !g.gelu_grad && g.dropout == nullptr && !g.b_mn_major && g.bn.x == nullptr && g.col_stats == nullptr && g.N % 256 == 0 &&
                    g.K >= 256 &&
                    (int64_t)((g.M + kBlockM - 1) / kBlockM) * (g.N / 256) >= kNumSMs;
  const int bn = n64 ? 64 : (wide ? 256 : 128);
  if (const char* e = tmap2d(&tmA, g.A, g.K, g.M, g.lda, kBlockK, kBlockM)) return e;
  if (!g.b_mn_major) {
    if (const char* e = tmap2d(&tmB, g.B, g.K, g.N, g.ldb, kBlockK, bn)) return e;
  } else {
    if (const char* e = tmap2d(&tmB, g.B, g.N, g.K, g.ldb, 64, kBlockK)) return e;
  }
  if (const char* e = tmap2d(&tmD, g.D, g.N, g.M, g.ldd, 64, kBlockM)) return e;
  PersistParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K;
  p.tiles_m = (g.M + kBlockM - 1) / kBlockM;
  p.tiles_n = (g.N + bn - 1) / bn;
  p.num_kb = (g.K + kBlockK - 1) / kBlockK;
  p.col_scale = g.col_scale; p.col_shift = g.col_shift; p.relu = g.relu ? 1 : 0;
  p.col_stats = g.col_stats;
  p.add_src = reinterpret_cast<const __nv_bfloat16*>(g.add_src);
  p.ld_add = g.ld_add;
  alignas(64) CUtensorMap tmAdd;
  const CUtensorMap* padd = nullptr;
  if (g.add_src != nullptr) {
    if (g.N % 8 != 0 || g.ld_add % 8 != 0 || (reinterpret_cast<uintptr_t>(g.add_src) & 15) != 0)
      return "gemm add_src needs N % 8 == 0 and 16-byte aligned rows";
    if (const char* e = tmap2d(&tmAdd, g.add_src, g.N, g.M, g.ld_add, 64, kBlockM)) return e;
    padd = &tmAdd;
  }
  if (g.dropout != nullptr) {
    if (g.b_mn_major || g.add_src == nullptr || g.gelu || g.gelu_grad || g.bn.x != nullptr || g.col_stats != nullptr ||
        g.relu || g.col_scale != nullptr)
      return "gemm residual-dropout epilogue: forward GEMM (B K-major) with an addend and an optional shift only";
    p.drop = *g.dropout;
    return n64 ? launch_p<64, 6, 0, 0, 0, 4>(tmA, tmB, tmD, p, stream, padd)
               : launch_p<128, 5, 0, 0, 0, 4>(tmA, tmB, tmD, p, stream, padd);
  }
  if (g.bn.x != nullptr) {
    // dgrad whose output is the gradient of a BatchNorm output: reduce it in the epilogue
    if (!g.b_mn_major || g.col_stats != nullptr) return "fused BN-backward reduction is a dgrad (B MN-major) feature";
    alignas(64) CUtensorMap tmBx, tmBy;
    if (const char* e = tmap2d(&tmBx, g.bn.x, g.N, g.M, g.ldd, 64, kBlockM)) return e;
    const bool has_y = g.bn.relu && g.bn.y != nullptr;
    const bool has_mask = g.bn.relu && g.bn.mask != nullptr;
    if (has_y && has_mask) return "fused BN-backward reduction: give the BN output or its mask bits, not both";
    if (has_y)
      if (const char* e = tmap2d(&tmBy, g.bn.y, g.N, g.M, g.ldd, 64, kBlockM)) return e;
    if (has_mask) {
      // uint8 [M, N / 8], one 16-byte box per 128-column tile
      if (g.N % 128 != 0) return "fused BN-backward reduction with mask bits needs N % 128 == 0";
      const uint64_t dims[2] = {(uint64_t)g.N / 8, (uint64_t)g.M};
      const uint64_t st[1] = {(uint64_t)g.N / 8};
      const uint32_t box[2] = {16, kBlockM};
      if (const char* e = encode_tmap_strided(&tmBy, g.bn.mask, 2, dims, st, box, nullptr, 1, 0)) return e;
    }
    fill_bn(p, g.bn);
    const CUtensorMap* pby = (has_y || has_mask) ? &tmBy : nullptr;
    return n64 ? launch_p<64, 4, 1, 2>(tmA, tmB, tmD, p, stream, padd, &tmBx, pby)
               : launch_p<128, 3, 1, 2>(tmA, tmB, tmD, p, stream, padd, &tmBx, pby);
  }
  if (g.gelu_grad) {
    if (!g.b_mn_major || g.add_src == nullptr || g.gelu || g.col_stats != nullptr || g.relu || g.col_scale != nullptr ||
        g.col_shift != nullptr)
      return "gemm GELU-gradient epilogue: dgrad GEMM (B MN-major) with u as the addend only";
    return n64 ? launch_p<64, 6, 1, 0, 0, 3>(tmA, tmB, tmD, p, stream, padd)
               : launch_p<128, 5, 1, 0, 0, 3>(tmA, tmB, tmD, p, stream, padd);
  }
  if (g.gelu) {
    if (g.b_mn_major || g.add_src != nullptr || g.col_stats != nullptr || g.relu)
      return "gemm GELU epilogue: forward GEMM (B K-major) with an optional scale / shift only";
    if (g.gelu_u != nullptr) {
      if (g.N % 8 != 0 || g.ld_u % 8 != 0 || (reinterpret_cast<uintptr_t>(g.gelu_u) & 15) != 0)
        return "gemm GELU epilogue: u needs N % 8 == 0 and 16-byte aligned rows";
      p.aux = reinterpret_cast<__nv_bfloat16*>(g.gelu_u);
      p.ld_aux = g.ld_u;
      return n64 ? launch_p<64, 6, 0, 0, 0, 2>(tmA, tmB, tmD, p, stream) : launch_p<128, 5, 0, 0, 0, 2>(tmA, tmB, tmD, p, stream);
    }
    return n64 ? launch_p<64, 6, 0, 0, 0, 1>(tmA, tmB, tmD, p, stream) : launch_p<128, 5, 0, 0, 0, 1>(tmA, tmB, tmD, p, stream);
  }
  if (!g.b_mn_major) {
    if (wide) return launch_p<256, 3, 0>(tmA, tmB, tmD, p, stream, padd);
    return n64 ? launch_p<64, 6, 0>(tmA, tmB, tmD, p, stream, padd) : launch_p<128, 5, 0>(tmA, tmB, tmD, p, stream, padd);
  }
  return n64 ? launch_p<64, 6, 1>(tmA, tmB, tmD, p, stream, padd) : launch_p<128, 5, 1>(tmA, tmB, tmD, p, stream, padd);
}

// conv front end: geometry comes from conv3x3.cu's planner
const char* conv3x3_bf16_persistent(const Conv3x3Args& a, int BH, int BN, int tiles_h, int tiles_img,
                                    cudaStream_t stream) {
  const bool dg = a.dgrad;
  const int cx = dg ? a.Cout : a.Cin, cy = dg ? a.Cin : a.Cout;
  const int groups = dg ? 1 : a.groups;
  const int cin_g = cx / groups, cout_g = cy / groups;
  const bool n64 = cout_g <= 64;
  const int bn = n64 ? 64 : 128;
  alignas(64) CUtensorMap tmX, tmW, tmY;
  const int sd = a.stride == 2 ? 2 : 1;
  if (sd == 2 && (dg || 2 * a.W > 256 || 2 * BH > 256)) return "conv3x3 stride 2: fprop only, output width <= 128";
  // 1x1 / pad 0 / stride 2: the centre tap of the stride-2 3x3 -- the same strided input map, one tap at (0, 0)
  const bool k1 = a.ksize == 1;
  if (k1 && (sd != 2 || groups != 1)) return "conv1x1 stride 2: dense, stride 2 only";
  const int taps = k1 ? 1 : 9;
  const bool halo = g_conv_halo && sd == 1 &&
                    halo_geometry(a.N, a.H, a.W, &BH, &BN, &tiles_h, &tiles_img);
  if (halo) {
    const uint64_t dims[4] = {(uint64_t)cx, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cx * 2, (uint64_t)a.W * cx * 2, (uint64_t)a.H * a.W * cx * 2};
    const uint32_t box[4] = {64, (uint32_t)(a.W + 1), (uint32_t)BH, (uint32_t)BN};
    if (const char* e = encode_tmap_bf16(&tmX, a.X, 4, dims, st, box)) return e;
  } else {
    // stride 2: the input is [N, 2H, 2W, C]; a box that spans 2W x 2BH elements with traversal stride 2 in w and h
    // delivers the W x BH pixels a filter tap needs, starting at column s - 1 and row 2*h0 + r - 1
    const uint64_t dims[4] = {(uint64_t)cx, (uint64_t)a.W * sd, (uint64_t)a.H * sd, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cx * 2, (uint64_t)a.W * sd * cx * 2, (uint64_t)a.H * sd * a.W * sd * cx * 2};
    const uint32_t box[4] = {64, (uint32_t)(a.W * sd), (uint32_t)(BH * sd), (uint32_t)BN};
    const uint32_t es[4] = {1, (uint32_t)sd, (uint32_t)sd, 1};
    if (const char* e = encode_tmap_strided(&tmX, a.X, 4, dims, st, box, es, 2)) return e;
  }
  {
    const uint64_t dims[4] = {(uint64_t)cy, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cy * 2, (uint64_t)a.W * cy * 2, (uint64_t)a.H * a.W * cy * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)BH, (uint32_t)BN};
    if (const char* e = encode_tmap_bf16(&tmY, a.Y, 4, dims, st, box)) return e;
  }
  const int w_cin = a.Cin / a.groups;      // channel extent of the KRSC weight tensor
  if (const char* e = tmap2d(&tmW, a.Wt, (uint64_t)taps * w_cin, a.Cout, (uint64_t)taps * w_cin, 64, dg ? kBlockK : bn))
    return e;
  PersistParams p{};
  p.M = tiles_img * tiles_h * kBlockM; p.N = cy; p.K = taps * cx;
  p.tiles_m = tiles_img * tiles_h;
  p.tiles_n = (cy + bn - 1) / bn;
  p.kc_blocks = cin_g / kBlockK;
  p.num_kb = (halo ? 3 : taps) * p.kc_blocks;
  if (k1) {
    p.ntaps = 1;
    p.tap_dh[0] = p.tap_dw[0] = p.tap_w[0] = 0;
  }
  p.Wb = halo ? a.W + 1 : a.W;
  p.b_res = (halo && n64 && p.kc_blocks == 1 && g_conv_bres) ? 1 : 0;
  p.col_stats = dg ? nullptr : a.col_stats;
  p.col_scale = dg ? nullptr : a.col_scale;
  p.col_shift = dg ? nullptr : a.col_shift;
  p.relu = (!dg && a.relu) ? 1 : 0;
  p.cin_g = cin_g; p.cout_g = cout_g;
  p.n_img = a.N; p.H = a.H; p.W = a.W; p.c_in_w = w_cin; p.BH = BH; p.BN = BN; p.tiles_h = tiles_h;
  p.stride = sd;
  if (dg && a.bn.x != nullptr) {
    if (a.bn.mask != nullptr) return "fused BN-backward reduction with mask bits is a 1x1 dgrad feature";
    alignas(64) CUtensorMap tmBx, tmBy;
    const uint64_t dims[4] = {(uint64_t)cy, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {(uint64_t)cy * 2, (uint64_t)a.W * cy * 2, (uint64_t)a.H * a.W * cy * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)BH, (uint32_t)BN};
    if (const char* e = encode_tmap_bf16(&tmBx, a.bn.x, 4, dims, st, box)) return e;
    const bool has_y = a.bn.relu && a.bn.y != nullptr;
    if (has_y)
      if (const char* e = encode_tmap_bf16(&tmBy, a.bn.y, 4, dims, st, box)) return e;
    fill_bn(p, a.bn);
    if (halo)
      return n64 ? launch_p<64, 9, 3, 2, 3>(tmX, tmW, tmY, p, stream, nullptr, &tmBx, has_y ? &tmBy : nullptr)
                 : launch_p<128, 4, 3, 2, 2>(tmX, tmW, tmY, p, stream, nullptr, &tmBx, has_y ? &tmBy : nullptr);
    return n64 ? launch_p<64, 4, 3, 2>(tmX, tmW, tmY, p, stream, nullptr, &tmBx, has_y ? &tmBy : nullptr)
               : launch_p<128, 3, 3, 2>(tmX, tmW, tmY, p, stream, nullptr, &tmBx, has_y ? &tmBy : nullptr);
  }
  if (halo) {
    // 64-column tiles: six A slots (with resident weights the A ring is all that is in flight, and L2 -> SM throughput is
    // bytes in flight over the load latency)
    if (!dg)
      return n64 ? launch_p<64, 9, 2, 0, 6>(tmX, tmW, tmY, p, stream) : launch_p<128, 7, 2, 0, 3>(tmX, tmW, tmY, p, stream);
    return n64 ? launch_p<64, 9, 3, 0, 6>(tmX, tmW, tmY, p, stream) : launch_p<128, 7, 3, 0, 3>(tmX, tmW, tmY, p, stream);
  }
  if (!dg) return n64 ? launch_p<64, 6, 2>(tmX, tmW, tmY, p, stream) : launch_p<128, 5, 2>(tmX, tmW, tmY, p, stream);
  return n64 ? launch_p<64, 6, 3>(tmX, tmW, tmY, p, stream) : launch_p<128, 5, 3>(tmX, tmW, tmY, p, stream);
}

void set_epilogue_warps(int n) { g_epi16 = n >= 16; }
void set_persist_trace(long long* buf) { g_trace = buf; }
// the tile geometry of the halo layout, for the CPU replay of its index math (tests/test_halo_plan_cpu.py)
bool conv3x3_halo_plan(int N, int H, int W, int* BH, int* BN, int* tiles_h, int* tiles_img) {
  return halo_geometry(N, H, W, BH, BN, tiles_h, tiles_img);
}
void set_conv_halo(bool on) { g_conv_halo = on; }
void set_conv_resident_weights(bool on) { g_conv_bres = on; }
bool get_conv_halo() { return g_conv_halo; }

namespace {
// One parity class (ph, pw) of a stride-2 input gradient: a stride-1 dgrad-mode launch over dY with the taps of that class,
// storing the pixels (2 i + ph, 2 j + pw) of dX through a tensor map with doubled pixel strides.  tmX / tmW are the dY
// and weight maps, c_in_w the weight's channel extent per tap (Cin), taps {dh, dw, weight tap} of the class.
const char* dgrad_s2_parity(const Conv3x3Args& a, int BH, int BN, int tiles_h, int tiles_img, const CUtensorMap& tmX,
                            const CUtensorMap& tmW, int ph, int pw, int ntaps, const signed char (*taps)[3],
                            cudaStream_t stream) {
  const int cx = a.Cout, cy = a.Cin;
  const bool n64 = cy <= 64;
  const int bn = n64 ? 64 : 128;
  const uint64_t W2 = 2ull * a.W, H2 = 2ull * a.H;
  alignas(64) CUtensorMap tmY;
  {
    // the pixels (2 i + ph, 2 j + pw) of dX as a dense-looking [N, Ho, Wo, Cin] tensor with doubled pixel strides
    const uint64_t dims[4] = {(uint64_t)cy, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
    const uint64_t st[3] = {2ull * cy * 2, 2ull * W2 * cy * 2, H2 * W2 * cy * 2};
    const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)BH, (uint32_t)BN};
    const char* base = reinterpret_cast<const char*>(a.Y) + ((uint64_t)ph * W2 + pw) * cy * 2;
    if (const char* e = encode_tmap_bf16(&tmY, base, 4, dims, st, box)) return e;
  }
  PersistParams p{};
  p.M = tiles_img * tiles_h * kBlockM; p.N = cy; p.K = ntaps * cx;
  p.tiles_m = tiles_img * tiles_h;
  p.tiles_n = (cy + bn - 1) / bn;
  p.kc_blocks = cx / kBlockK;
  p.cin_g = cx; p.cout_g = cy;
  p.n_img = a.N; p.H = a.H; p.W = a.W; p.c_in_w = a.Cin; p.BH = BH; p.BN = BN; p.tiles_h = tiles_h;
  p.stride = 1;
  for (int t = 0; t < ntaps; ++t) {
    p.tap_dh[t] = taps[t][0];
    p.tap_dw[t] = taps[t][1];
    p.tap_w[t] = taps[t][2];
  }
  p.ntaps = ntaps;
  p.num_kb = ntaps * p.kc_blocks;
  return n64 ? launch_p<64, 6, 3>(tmX, tmW, tmY, p, stream) : launch_p<128, 5, 3>(tmX, tmW, tmY, p, stream);
}

// dY [N, Ho, Wo, Cout] as the A operand of the dgrad mode
const char* dgrad_s2_dy_map(const Conv3x3Args& a, int BH, int BN, CUtensorMap* tmX) {
  const int cx = a.Cout;
  const uint64_t dims[4] = {(uint64_t)cx, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.N};
  const uint64_t st[3] = {(uint64_t)cx * 2, (uint64_t)a.W * cx * 2, (uint64_t)a.H * a.W * cx * 2};
  const uint32_t box[4] = {64, (uint32_t)a.W, (uint32_t)BH, (uint32_t)BN};
  return encode_tmap_bf16(tmX, a.X, 4, dims, st, box);
}
}  // namespace

// Input gradient of the 3x3 / pad 1 / STRIDE 2 convolution (round 2).  dX[n, h, w] = sum over the taps (r, s) with
// h + 1 - r and w + 1 - s even of dY[n, (h + 1 - r) / 2, (w + 1 - s) / 2] * W[:, r, s, :]: for a fixed parity (h & 1, w & 1)
// that is a stride-1 convolution of dY with 1, 2, 2 or 4 taps whose result lands on every second pixel of dX.  Four
// launches of the dgrad mode with an explicit tap list and a strided output tensor map -- 9 tap-MMAs per output-gradient
// pixel in total, exactly the work of the forward pass (zero-insertion + stride-1 dgrad costs four times that).
// a.X = dY [N, Ho, Wo, Cout], a.Y = dX [N, 2 Ho, 2 Wo, Cin], a.N / H / W = the dY geometry.
const char* conv3x3_dgrad_s2_persistent(const Conv3x3Args& a, int BH, int BN, int tiles_h, int tiles_img,
                                        cudaStream_t stream) {
  alignas(64) CUtensorMap tmX, tmW;
  if (const char* e = dgrad_s2_dy_map(a, BH, BN, &tmX)) return e;
  if (const char* e = tmap2d(&tmW, a.Wt, (uint64_t)9 * a.Cin, a.Cout, (uint64_t)9 * a.Cin, 64, kBlockK)) return e;
  for (int ph = 0; ph < 2; ++ph) {
    for (int pw = 0; pw < 2; ++pw) {
      signed char taps[4][3];
      int nt = 0;
      for (int r = 0; r < 3; ++r) {
        if (((ph + 1 - r) & 1) != 0) continue;
        for (int sft = 0; sft < 3; ++sft) {
          if (((pw + 1 - sft) & 1) != 0) continue;
          taps[nt][0] = (signed char)((ph + 1 - r) / 2);      // exact: the numerator is even (0 or 2)
          taps[nt][1] = (signed char)((pw + 1 - sft) / 2);
          taps[nt][2] = (signed char)(r * 3 + sft);
          ++nt;
        }
      }
      if (const char* e = dgrad_s2_parity(a, BH, BN, tiles_h, tiles_img, tmX, tmW, ph, pw, nt, taps, stream)) return e;
    }
  }
  return nullptr;
}

// Input gradient of the 1x1 / pad 0 / stride 2 convolution: dX[n, 2h, 2w] = dY[n, h, w] * W and zero elsewhere.  dX is
// zero-filled (a memset node when captured in a graph), then ONE dgrad-mode launch with the single tap (0, 0) stores the
// even-even pixels through the parity-(0, 0) map of the 3x3 path.  dX stays a dense tensor, so a consumer that adds it to
// another gradient (the bottleneck's forked input) reads it like any other.  Weight [Cout, Cin], read MN-major.
const char* conv1x1_dgrad_s2_persistent(const Conv3x3Args& a, int BH, int BN, int tiles_h, int tiles_img,
                                        cudaStream_t stream) {
  alignas(64) CUtensorMap tmX, tmW;
  if (const char* e = dgrad_s2_dy_map(a, BH, BN, &tmX)) return e;
  if (const char* e = tmap2d(&tmW, a.Wt, (uint64_t)a.Cin, a.Cout, (uint64_t)a.Cin, 64, kBlockK)) return e;
  const size_t dx_bytes = (size_t)a.N * (2 * a.H) * (2 * a.W) * a.Cin * 2;
  cudaError_t ce = cudaMemsetAsync(a.Y, 0, dx_bytes, stream);
  if (ce != cudaSuccess) return cudaGetErrorString(ce);
  const signed char centre[1][3] = {{0, 0, 0}};
  return dgrad_s2_parity(a, BH, BN, tiles_h, tiles_img, tmX, tmW, 0, 0, 1, centre, stream);
}

}  // namespace edl
