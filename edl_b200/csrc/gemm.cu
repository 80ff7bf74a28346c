// wgmma / TMA GEMM for sm_90a with fused epilogues (SURVEY K1, K5 and the conv-as-GEMM
// half of K2).  The reference gets these from cuDNN/cuBLAS via Paddle
// (example/distill/resnet/models/resnet_vd.py:153-162 conv2d, :135-141 fc); this is an
// independent Hopper-native implementation.
//
//   D[M,N] = A[M,K] * B[N,K]^T          (NHWC 1x1 conv fwd, FC)      A K-major,  B K-major
//   D[M,N] = A[M,K] * B[K,N]            (1x1 conv dgrad)             A K-major,  B MN-major
//   D[M,N] = A[K,M]^T * B[K,N]          (1x1 conv wgrad, split-K)    A MN-major, B MN-major
//
// Structure (one CTA per 128 x BLOCK_N output tile):
//   warp 0      : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx)
//   warps 4..11 : two consumer warpgroups, each owns 64 rows of the tile: wgmma.mma_async from the ring into fp32
//                 register accumulators, then the epilogue: per-channel scale/shift/ReLU ->
//                 bf16 -> swizzled smem -> TMA store; per-channel sum / sum^2 of the stored values
//                 (train-mode BatchNorm statistics) reduced from the staged tile and pushed with
//                 fp32 atomics, so BN needs no extra pass over the conv output.
//                 Weight-gradient variant (EPI 1): coalesced bf16 stores, or fp32 partial tiles per K split
//                 that splitk_reduce_kernel sums.
#include <cuda.h>
#include <cstdio>
#include <mutex>

#include "gemm.h"
#include "kernels.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = one 128-byte swizzle span
constexpr int MMA_K = 16;
constexpr int kGemmThreads = 384;   // producer warpgroup (one warp works) + two consumer warpgroups
constexpr int kEpiThreads = 256;

struct GemmParams {
  int M, N, K;
  int kb_per_split;
  const float* col_scale;
  const float* col_shift;
  int relu;
  float* col_stats;  // [2N]
  __nv_bfloat16* out_bf16;   // EPI 1: bf16 [M, n_out], row pitch ldo (+= when accumulate)
  long long ldo;
  int n_out;                 // EPI 1: columns stored (<= N; the rest of B's width is padding)
  int accumulate;
  float* part;       // EPI 1 with a K split: partial tiles [split][tiles][BLOCK_M x BLOCK_N]
  // GEMM -> peer ship (see gemm.h)
  uint32_t* ship_flag;
  const uint32_t* ship_seq_ptr;
  uint32_t ship_seq_imm;
  unsigned int* ship_done;
};

template <int BLOCK_N, int STAGES>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kDBytes = BLOCK_M * BLOCK_N * 2;
  static constexpr int kTileBytes =
      STAGES * kStageBytes > kDBytes ? STAGES * kStageBytes : kDBytes;
  static constexpr int kBarOffset = kTileBytes;
  static constexpr int kTotal = kTileBytes + 256 + 1024;  // barriers + alignment slack
};

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmD, const GemmParams p) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int tile = blockIdx.x;
  const int m0 = (tile / tiles_n) * BLOCK_M;
  const int n0 = (tile % tiles_n) * BLOCK_N;
  const int total_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  int kb_end = kb_begin + p.kb_per_split;
  if (kb_end > total_kb) kb_end = total_kb;
  const int num_kb = kb_end - kb_begin;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (EPI == 0) ptx::prefetch_tmap(&tmD);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (num_kb > 0) {
    if (warp == 0) {
      // ------------------------------------------------------------ TMA producer
      // warp-uniform loop, one elected lane issues (see gemm_persist.cu: loops under `if (lane == 0)` cost a vote +
      // broadcast sequence per uniform-register operand)
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        ptx::mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * L::kStageBytes;
        uint8_t* sb = sa + L::kABytes;
        const int k0 = (kb_begin + i) * BLOCK_K;
        if (ptx::elect_one()) {
          ptx::mbar_arrive_expect_tx(&full_bar[s], L::kStageBytes);
          if (!A_MN) {
            ptx::tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);
          } else {
#pragma unroll
            for (int h = 0; h < BLOCK_M / 64; ++h)
              ptx::tma_load_2d(sa + h * 8192, &tmA, &full_bar[s], m0 + h * 64, k0);
          }
          if (!B_MN) {
            ptx::tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);
          } else {
#pragma unroll
            for (int h = 0; h < BLOCK_N / 64; ++h)
              ptx::tma_load_2d(sb + h * 8192, &tmB, &full_bar[s], n0 + h * 64, k0);
          }
        }
        __syncwarp();
      }
    } else if (warp >= 4) {
      // ------------------------------------------------------------ consumers: MMA, then epilogue (warps 4..11)
      const int cw = (warp - 4) >> 2;                       // consumer warpgroup = 64-row half of the tile
      const int et = threadIdx.x - 128;                     // 0..255 epilogue thread id
      const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // first accumulator row of this thread (second: + 8)
      const int cq = (lane & 3) * 2;                        // column of the thread inside an 8-column group
      float acc[BLOCK_N / 2];
      using Mma = ptx::WgmmaBf16<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>;
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        ptx::mbar_wait(&full_bar[s], (i / STAGES) & 1);
        const uint32_t sa = ptx::smem_u32(smem + s * L::kStageBytes) + cw * 8192;   // 64 rows (or 64 MN elements) per group
        const uint32_t sb = ptx::smem_u32(smem + s * L::kStageBytes) + L::kABytes;
        // a k step adds 32 bytes (K-major) or 2048 bytes (MN-major) to the start address field, which counts 16-byte units
        const uint64_t da0 = A_MN ? ptx::make_smem_desc(sa, 8192, 1024) : ptx::make_smem_desc(sa, 16, 1024);
        const uint64_t db0 = B_MN ? ptx::make_smem_desc(sb, 8192, 1024) : ptx::make_smem_desc(sb, 16, 1024);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          Mma::mma(acc, da0 + (uint64_t)(k * (A_MN ? 128 : 2)), db0 + (uint64_t)(k * (B_MN ? 128 : 2)), (i | k) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        // the MMAs of the previous k-block have read their stage: hand it back to the producer
        ptx::wgmma_wait<1>();
        if (i > 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[(i - 1) % STAGES]);
      }
      ptx::wgmma_wait<0>();
      asm volatile("bar.sync 1, 256;" ::: "memory");       // both groups are done reading the ring: it becomes the staging tile
      if (EPI == 0) {
        uint8_t* sd = smem;  // pipeline stages are drained: reuse them as the store staging tile
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = n0 + j * 8 + cq;
          float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
          if (p.col_scale != nullptr) {
            const float s0 = col < p.N ? p.col_scale[col] : 0.f, s1 = col + 1 < p.N ? p.col_scale[col + 1] : 0.f;
            v0 *= s0; v1 *= s1; v2 *= s0; v3 *= s1;
          }
          if (p.col_shift != nullptr) {
            const float s0 = col < p.N ? p.col_shift[col] : 0.f, s1 = col + 1 < p.N ? p.col_shift[col + 1] : 0.f;
            v0 += s0; v1 += s1; v2 += s0; v3 += s1;
          }
          if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
          // staging tile: 64-column halves of [BLOCK_M rows][128 B], 16-byte chunks XOR-swizzled by the row (= what TMA expects)
          uint8_t* hp = sd + (j >> 3) * (BLOCK_M * 128) + cq * 2;
          *reinterpret_cast<__nv_bfloat162*>(hp + row * 128 + (((j & 7) ^ (row & 7)) << 4)) = __floats2bfloat162_rn(v0, v1);
          *reinterpret_cast<__nv_bfloat162*>(hp + (row + 8) * 128 + (((j & 7) ^ ((row + 8) & 7)) << 4)) = __floats2bfloat162_rn(v2, v3);
        }
        ptx::fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (et == 0) {
#pragma unroll
          for (int h = 0; h < (BLOCK_N + 63) / 64; ++h)
            if (n0 + h * 64 < p.N) ptx::tma_store_2d(&tmD, sd + h * (BLOCK_M * 128), n0 + h * 64, m0);
          ptx::tma_store_commit();
        }
        if (p.col_stats != nullptr) {
          int rows_valid = p.M - m0;
          if (rows_valid > BLOCK_M) rows_valid = BLOCK_M;
          for (int col = et; col < BLOCK_N; col += kEpiThreads) {
            const bool valid = n0 + col < p.N;     // no early exit: the whole warp shuffles below
            const int half = col >> 6, cc = col & 63, chunk = cc >> 3, within = cc & 7;
            const uint8_t* base = sd + half * (BLOCK_M * 128) + within * 2;
            float s = 0.f, sq = 0.f;
#pragma unroll 8
            for (int rr = 0; rr < (valid ? rows_valid : 0); ++rr) {
              const __nv_bfloat16 hv = *reinterpret_cast<const __nv_bfloat16*>(
                  base + rr * 128 + ((chunk ^ (rr & 7)) << 4));
              const float v = __bfloat162float(hv);
              s += v;
              sq = fmaf(v, v, sq);
            }
            // four neighbouring columns -> one vector reduction (lane 4i collects lanes 4i..4i+3)
            const float s1 = __shfl_down_sync(0xffffffffu, s, 1), s2 = __shfl_down_sync(0xffffffffu, s, 2),
                        s3 = __shfl_down_sync(0xffffffffu, s, 3);
            const float q1 = __shfl_down_sync(0xffffffffu, sq, 1), q2 = __shfl_down_sync(0xffffffffu, sq, 2),
                        q3 = __shfl_down_sync(0xffffffffu, sq, 3);
            float* ps = &p.col_stats[n0 + col];
            float* pq = &p.col_stats[p.N + n0 + col];
            const int c4 = col & ~3;   // the decision is per group of four columns, identical in its 4 lanes
            const bool vec = (p.N % 4 == 0) && n0 + c4 + 3 < p.N &&
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
        if (et == 0) {
          if (p.ship_flag == nullptr) {
            ptx::tma_store_wait_read0();
          } else {
            // the tile went to a peer GPU: wait until the bulk store has fully completed (not just
            // read its smem source), order it system-wide, count this CTA in; the last one raises
            // the consumer's flag.
            ptx::tma_store_wait0();
            __threadfence_system();
            const unsigned int prev = atomicAdd(p.ship_done, 1u);
            if (prev == gridDim.x - 1) {
              *p.ship_done = 0u;
              __threadfence_system();
              const uint32_t seq = p.ship_seq_ptr != nullptr ? *p.ship_seq_ptr : p.ship_seq_imm;
              asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p.ship_flag), "r"(seq) : "memory");
            }
          }
        }
      } else {
        // weight gradient: stage the fp32 tile in smem (the pipeline stages are drained), then store it COALESCED:
        // consecutive threads cover consecutive 16-byte pieces of a row.  Without a K split this CTA owns the tile and
        // writes bf16 (+= when accumulating); with one it stores its partial tile for splitk_reduce_kernel.
        constexpr int kPitch = BLOCK_N * 4 + 32;        // bytes; +32 spreads the eight rows of a warp's store over the banks
        constexpr int kVecPerRow = BLOCK_N / 4;         // float4 per row
        uint8_t* sf = smem;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(sf + row * kPitch + (j * 8 + cq) * 4) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(sf + (row + 8) * kPitch + (j * 8 + cq) * 4) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (gridDim.z == 1) {
          int rows_valid = p.M - m0;
          if (rows_valid > BLOCK_M) rows_valid = BLOCK_M;
          int cols_valid = p.n_out - n0;
          if (cols_valid > BLOCK_N) cols_valid = BLOCK_N;
          // 8-byte stores need 4-column aligned rows; an output narrower than B (n_out % 4 != 0) is stored per element
          const bool vec = (p.ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out_bf16) & 7) == 0;
          for (int f = et; f < rows_valid * kVecPerRow; f += kEpiThreads) {
            const int rr = f / kVecPerRow, c4 = (f % kVecPerRow) * 4;
            if (c4 >= cols_valid) continue;
            const float4 t = *reinterpret_cast<const float4*>(sf + rr * kPitch + c4 * 4);
            __nv_bfloat16* dst = p.out_bf16 + (int64_t)(m0 + rr) * p.ldo + n0 + c4;
            if (vec && c4 + 3 < cols_valid) store_bf16x4(dst, t, p.accumulate);
            else store_bf16_tail(dst, t, cols_valid - c4, p.accumulate);
          }
        } else {
          float* dst = p.part + ((int64_t)blockIdx.z * gridDim.x + tile) * (BLOCK_M * BLOCK_N);
          for (int f = et; f < BLOCK_M * kVecPerRow; f += kEpiThreads) {
            const int rr = f / kVecPerRow, c4 = (f % kVecPerRow) * 4;
            *reinterpret_cast<float4*>(dst + rr * BLOCK_N + c4) = *reinterpret_cast<const float4*>(sf + rr * kPitch + c4 * 4);
          }
        }
      }
    }
  }
}

// -------------------------------------------------------------------------------------------
// host side

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

thread_local char g_tmap_err[256];

// 2-D bf16 tensor map: dims {inner, outer}, row pitch in elements, box {box_inner, box_outer}.
bool make_tmap_2d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t outer,
                  uint64_t pitch_elems, uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    snprintf(g_tmap_err, sizeof(g_tmap_err), "cuTensorMapEncodeTiled entry point not found");
    return false;
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    snprintf(g_tmap_err, sizeof(g_tmap_err),
             "cuTensorMapEncodeTiled failed: CUresult=%d ptr=%p dims={%llu,%llu} pitch=%llu box={%u,%u}",
             (int)r, ptr, (unsigned long long)inner, (unsigned long long)outer,
             (unsigned long long)pitch_elems, box_inner, box_outer);
  return r == CUDA_SUCCESS;
}

}  // namespace

// N-d bf16 tensor map (128B swizzle, zero OOB fill) for the other TMA kernels (conv3x3.cu).
// dims / box are innermost-first; strides_bytes has rank-1 entries (dims 1..rank-1).
const char* encode_tmap_bf16(void* out, const void* ptr, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_tmap(out, ptr, rank, dims, strides_bytes, box, 2);
}

const char* encode_tmap(void* out, const void* ptr, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes) {
  return encode_tmap_strided(out, ptr, rank, dims, strides_bytes, box, nullptr, elem_bytes);
}

// elem_strides (optional): traversal stride per dimension.  With stride t the unit loads ceil(box / t) elements
// along that dimension (every t-th one), i.e. box[i] = n * t selects n elements -- how a stride-2 convolution reads
// its input without an im2col or a subsampling pass.
const char* encode_tmap_strided(void* out, const void* ptr, int rank, const uint64_t* dims,
                                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                                int elem_bytes, bool swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return "cuTensorMapEncodeTiled entry point not found";
  cuuint64_t d[5], st[4];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; es[i] = elem_strides != nullptr ? elem_strides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(out),
                  elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank,
                  const_cast<void*>(ptr), d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(g_tmap_err, sizeof(g_tmap_err),
             "cuTensorMapEncodeTiled(rank %d) failed: CUresult=%d ptr=%p dims={%llu,%llu,..} box={%u,%u,..}",
             rank, (int)r, ptr, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return g_tmap_err;
  }
  return nullptr;
}

namespace {

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN, int EPI>
const char* launch_variant(const GemmArgs& g, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, STAGES>;
  CUtensorMap tmA, tmB, tmD;
  bool ok = true;
  // A: K-major -> global [M rows][K] ; MN-major -> global [K rows][M]
  if (!A_MN) ok &= make_tmap_2d(&tmA, g.A, g.K, g.M, g.lda, BLOCK_K, BLOCK_M);
  else ok &= make_tmap_2d(&tmA, g.A, g.M, g.K, g.lda, 64, BLOCK_K);
  if (!B_MN) ok &= make_tmap_2d(&tmB, g.B, g.K, g.N, g.ldb, BLOCK_K, BLOCK_N);
  else ok &= make_tmap_2d(&tmB, g.B, g.N, g.K, g.ldb, 64, BLOCK_K);
  if (EPI == 0) ok &= make_tmap_2d(&tmD, g.D, g.N, g.M, g.ldd, BLOCK_N < 64 ? BLOCK_N : 64, BLOCK_M);
  else tmD = tmA;
  if (!ok) return g_tmap_err;
  auto kern = gemm_wgmma_kernel<BLOCK_N, STAGES, A_MN, B_MN, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    apply_carveout((const void*)kern);
    attr_set = true;
  }
  GemmParams p;
  p.M = g.M; p.N = g.N; p.K = g.K;
  const int total_kb = (g.K + BLOCK_K - 1) / BLOCK_K;
  int split = EPI == 1 ? (g.split_k < 1 ? 1 : g.split_k) : 1;
  if (split > total_kb) split = total_kb;
  p.kb_per_split = (total_kb + split - 1) / split;
  split = (total_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.col_scale = g.col_scale;
  p.col_shift = g.col_shift;
  p.relu = g.relu ? 1 : 0;
  p.col_stats = g.col_stats;
  p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(g.D);
  p.ldo = g.ldd;
  p.n_out = (EPI == 1 && g.n_out > 0 && g.n_out < g.N) ? g.n_out : g.N;
  p.accumulate = g.accumulate ? 1 : 0;
  p.part = split > 1 ? g.partials : nullptr;
  p.ship_flag = EPI == 0 ? reinterpret_cast<uint32_t*>(g.ship_flag) : nullptr;
  p.ship_seq_ptr = reinterpret_cast<const uint32_t*>(g.ship_seq_ptr);
  p.ship_seq_imm = g.ship_seq_imm;
  p.ship_done = reinterpret_cast<unsigned int*>(g.ship_done);
  const int tiles_m = (g.M + BLOCK_M - 1) / BLOCK_M;
  const int tiles_n = (g.N + BLOCK_N - 1) / BLOCK_N;
  dim3 grid(tiles_m * tiles_n, 1, split);
  if (split > 1 && (g.partials == nullptr || g.partials_elems < (int64_t)split * grid.x * BLOCK_M * BLOCK_N))
    return "gemm_bf16: split_k > 1 needs a partial-tile buffer of split * tiles * 128 * BLOCK_N floats";
  kern<<<grid, kGemmThreads, L::kTotal, stream>>>(tmA, tmB, tmD, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cudaGetErrorString(e);
  if (split > 1) {
    splitk_reduce(g.partials, split, (int)grid.x, tiles_n, BLOCK_M, BLOCK_N, 1, 0, g.M, p.n_out, g.D, g.ldd,
                  g.accumulate, stream);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// Sum of the split-K partial tiles -> bf16 output (+= when accumulating).  A CTA of 256 threads covers 64 consecutive
// float4 of a tile row; its 4 thread groups each sum every 4th split (independent 16-byte loads, unrolled so that
// several are in flight), a shared-memory pass adds the 4 partial sums.  The kernel is latency-bound by construction
// (a few MB out of L2): the z-parallel layout keeps it at a few load latencies instead of split x load latency.
constexpr int kRedVec = 64;     // float4 per CTA

template <int kRedZ>            // split groups per CTA: 4, or 16 for deep splits (few tiles, 32+ partials each)
__global__ void __launch_bounds__(kRedVec * kRedZ)
splitk_reduce_kernel(const float* __restrict__ part, int split, int ctas, int tiles_n, int rows, int cols, int taps,
                     int cin, int M, int N, __nv_bfloat16* __restrict__ out, long long ldo, int accumulate) {
  __shared__ float4 sm[kRedZ][kRedVec];
  const int vec_per_row = cols / 4;
  const int64_t per_tile = (int64_t)rows * vec_per_row;
  const int64_t total = (int64_t)ctas * per_tile;
  const int64_t tile_elems = (int64_t)rows * cols;
  const int64_t zstride = (int64_t)ctas * tile_elems;
  const int vl = threadIdx.x % kRedVec, q = threadIdx.x / kRedVec;
  for (int64_t base = (int64_t)blockIdx.x * kRedVec; base < total; base += (int64_t)gridDim.x * kRedVec) {
    const int64_t i = base + vl;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    bool ok = i < total;
    int m = 0, n = 0;
    if (ok) {
      const int t = (int)(i / per_tile);
      const int rem = (int)(i - (int64_t)t * per_tile);
      const int rr = rem / vec_per_row, c4 = (rem - rr * vec_per_row) * 4;
      if (taps == 1) {
        m = (t / tiles_n) * rows + rr;
        n = (t % tiles_n) * cols + c4;
      } else {
        const int tile = t / 3, r = t - tile * 3, bn = cols / 3;
        const int s = c4 / bn, cc = c4 - s * bn;
        m = (tile / tiles_n) * rows + rr;
        n = (r * 3 + s) * cin + (tile % tiles_n) * bn + cc;
        ok = (tile % tiles_n) * bn + cc + 3 < cin;
      }
      ok = ok && m < M && n < N;
      if (ok) {
        const float* src = part + (int64_t)t * tile_elems + (int64_t)rr * cols + c4;
        int z = q;
        for (; z + 3 * kRedZ < split; z += 4 * kRedZ) {
          const float4 a = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)z * zstride));
          const float4 b = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)(z + kRedZ) * zstride));
          const float4 c = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)(z + 2 * kRedZ) * zstride));
          const float4 d = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)(z + 3 * kRedZ) * zstride));
          acc.x += (a.x + b.x) + (c.x + d.x); acc.y += (a.y + b.y) + (c.y + d.y);
          acc.z += (a.z + b.z) + (c.z + d.z); acc.w += (a.w + b.w) + (c.w + d.w);
        }
        for (; z < split; z += kRedZ) {
          const float4 a = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)z * zstride));
          acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
        }
      }
    }
    sm[q][vl] = acc;
    __syncthreads();
    if (q == 0 && ok) {
#pragma unroll
      for (int k = 1; k < kRedZ; ++k) {
        const float4 o = sm[k][vl];
        acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
      }
      // 8-byte stores need 4-column aligned rows; a row pitch or width that is not a multiple of 4 is stored per element
      const bool vec = (ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0 && n + 3 < N;
      if (vec) store_bf16x4(out + (int64_t)m * ldo + n, acc, accumulate);
      else store_bf16_tail(out + (int64_t)m * ldo + n, acc, N - n, accumulate);
    }
    __syncthreads();
  }
}

}  // namespace

void splitk_reduce(const float* partials, int split, int ctas, int tiles_n, int rows, int cols, int taps, int cin, int M,
                   int N, void* out_bf16, int64_t ldo, bool accumulate, cudaStream_t stream) {
  const int64_t total = (int64_t)ctas * rows * (cols / 4);
  int blocks = (int)((total + kRedVec - 1) / kRedVec);
  if (blocks < 1) blocks = 1;
  auto* out = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  if (split >= 32) {
    if (blocks > kNumSMs * 2) blocks = kNumSMs * 2;
    splitk_reduce_kernel<16><<<blocks, kRedVec * 16, 0, stream>>>(partials, split, ctas, tiles_n, rows, cols, taps, cin,
                                                                 M, N, out, (long long)ldo, accumulate ? 1 : 0);
  } else {
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    splitk_reduce_kernel<4><<<blocks, kRedVec * 4, 0, stream>>>(partials, split, ctas, tiles_n, rows, cols, taps, cin, M,
                                                               N, out, (long long)ldo, accumulate ? 1 : 0);
  }
}

const char* gemm_bf16(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return "empty GEMM";
  // cuTensorMapEncodeTiled is a driver call and needs a current context on THIS thread.  Autograd
  // worker threads may not have one yet (torch binds lazily; observed CUDA_ERROR_INVALID_CONTEXT
  // = 201 when a dgrad GEMM was the first CUDA work of the backward thread).
  if (g.device >= 0) {
    cudaError_t e = cudaSetDevice(g.device);
    if (e != cudaSuccess) return cudaGetErrorString(e);
  }
  const bool n64 = g.N <= 64;
  if (!g.a_mn_major && g.ship_flag == nullptr && persistent_gemm_enabled()) return gemm_bf16_persistent(g, stream);
  if (g.add_src != nullptr) return "gemm add_src is implemented by the persistent kernel only";
  if (g.gelu || g.gelu_grad) return "gemm GELU epilogue is implemented by the persistent kernel only";
  if (g.a_mn_major && g.b_mn_major)   // weight gradient
    return n64 ? launch_variant<64, 4, true, true, 1>(g, stream) : launch_variant<128, 3, true, true, 1>(g, stream);
  if (!g.a_mn_major && !g.b_mn_major)
    return n64 ? launch_variant<64, 4, false, false, 0>(g, stream)
               : launch_variant<128, 3, false, false, 0>(g, stream);
  if (!g.a_mn_major && g.b_mn_major)
    return n64 ? launch_variant<64, 4, false, true, 0>(g, stream)
               : launch_variant<128, 3, false, true, 0>(g, stream);
  return "unsupported operand layout";
}

}  // namespace edl
