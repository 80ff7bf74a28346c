// Bidirectional single-layer LSTM recurrence for sm_90a (the BiLSTM student of the NLP distillation), H = 128.
//
// Semantics are torch.nn.LSTM(batch_first=True, bidirectional=True) on right-padded sequences with per-sample lengths
// (pack_padded_sequence, enforce_sorted=False): gate order i, f, g, o; zero initial state; direction 0 runs sample b
// over t = 0 .. len_b - 1, direction 1 over t = len_b - 1 .. 0.  Lengths are clamped to [0, L] here (no host check).
// Step s of a direction reads time t(s) = s (forward) or len_b - 1 - s (reverse); a row with s >= len_b is inactive:
// its state is not updated, nothing of it is read (masking is by selection, so NaN in a padded row reaches nothing),
// and its outputs at time s are 0.
//
// Layout (time-major, row t * B + b):
//   xproj  bf16 [L * B, 8H]   X W_ih^T + b_ih + b_hh of both directions (one gemm_bf16), columns of direction d at
//                             d * 4H in the "thread order" below
//   hs     bf16 [(L + 2) * B, 2H]   h_t of direction d at row (t + 1) * B + b, columns d * H; blocks 0 and L + 1 are
//                             zero, so h_{t-1} of both directions is a plain view (the weight gradient of W_hh)
//   hn     bf16 [2, B, H]     final states (0 for a sample of length 0)
//   gates  bf16 [L * B, 2, H, 4]  post-activation (i, f, g, o) per unit, saved for the backward
//   cs     fp32 [L * B, 2, H]     cell state c_t, saved for the backward
//   dgates bf16 [L * B, 8H]   backward output in nn.LSTM's row order (d * 4H + gate * H + unit), 0 past the length
// gates / cs are written for active (b, t) only; hs and dgates are written everywhere.
//
// Forward: grid (2 directions, ceil(B / 64)), 256 threads = two consumer warpgroups.  Each CTA loads its direction's
// W_hh (4H x H bf16 = 128 KB) into shared memory once, with its rows permuted so that every accumulator thread holds
// all four gates of its hidden units: the wgmma fragment gives a thread the column pairs {8j + 2q, 8j + 2q + 1}
// (q = lane % 4); permuted row n = 16m + 8c + 2q + e of warpgroup w's 256 columns is gate 2c + e of unit
// 64w + 4m + q, so chunk 2m holds (i, f) and chunk 2m + 1 holds (g, o) of the units 64w + 4m + q.  Per step,
// acc = xproj row (loaded straight into the accumulator registers, then h_{t-1} W_hh^T is accumulated on top by
// 2 x 4 wgmma m64n256k16 per warpgroup); the gate nonlinearities and the c / h update run in those registers, c stays
// in 32 fp32 registers per thread, and h_t goes to the other of two 16 KB K-major A tiles (one bar.sync per step).
// xproj's "thread order" puts a thread's 64 values of a row at column w * 256 + q * 64 (eight 16-byte loads per row):
// column w * 256 + q * 64 + 4m + gate is gate `gate` of unit 64w + 4m + q.  These loads are issued right after the
// cell update of the previous step, so their latency overlaps the h store and the barrier.  (The reverse direction
// reads row b at t = len_b - 1 - s: each row is its own gather.)
//
// Backward: same grid.  Steps run from the tile's longest length down to 0.  dgates_{s+1} (64 x 4H bf16 = 64 KB,
// K-major, in the permuted order) and W_hh (the same 128 KB image, read as an MN-major B operand) are resident;
// dh = dY[t] (+ dh_n at the sample's last step) + dgates_{s+1} W_hh by 32 wgmma m64n64k16 per warpgroup (K = 4H,
// each warpgroup 64 of the H columns); dc is carried in fp32 registers; dgates_t is written to global memory in
// nn.LSTM order and, after a barrier that retires the step's reads, into the A tile.  Saved for the backward: the
// post-activation gates in bf16 and c in fp32 (tanh(c_t) is recomputed); the backward uses exactly these values.
//
// Activations: sigma(x) = __fdividef(1, 1 + __expf(-x)), tanh(x) = 2 sigma(2x) - 1 (CUDA C Programming Guide, intrinsic
// functions: __expf within 2 + floor(|1.173 x|) ulp, __fdividef within 2 ulp).
//
// Budget (ptxas -v, sm_90a, CUDA 12.9): forward 249 registers, backward 244 registers, no spills, no stack; dynamic shared memory:
// forward 128 KB W_hh + 2 x 16 KB h tiles + 256 B lengths + 1 KB alignment slack = 164,096 B; backward 128 KB
// W_hh + 64 KB dgates tile + 256 B + 1 KB = 197,888 B.  One CTA per SM; 2 * ceil(B / 64) CTAs: the recurrence is
// latency-bound and small batches leave most SMs idle.  No atomics (bitwise deterministic), no host synchronisation,
// no allocation: the launch can be captured in a CUDA graph.
#include "kernels.h"
#include "ptx.cuh"

namespace edl {
namespace {

constexpr int kH = kLstmHidden;
constexpr int kG = 4 * kH;                                  // gate rows per direction
constexpr int kRows = 64;                                   // batch rows per CTA
constexpr int kThreads = 256;
constexpr int kWBytes = kG * kH * 2;                        // 128 KB
constexpr int kHTile = kRows * kH * 2;                      // 16 KB
constexpr int kDgTile = kRows * kG * 2;                     // 64 KB
constexpr int kFwdSmem = kWBytes + 2 * kHTile + 256 + 1024;
constexpr int kBwdSmem = kWBytes + kDgTile + 256 + 1024;

// Byte offset of (row, k) in a K-major, 128B-swizzled tile of `rows` rows: 64-column slabs of rows x 128 B.
EDL_DEVICE uint32_t swz(int row, int k, int rows) {
  return (uint32_t)((k >> 6) * rows * 128 + row * 128 + ((((k & 63) >> 3) ^ (row & 7)) << 4) + (k & 7) * 2);
}

// nn.LSTM row of permuted gate row p (see the header)
EDL_DEVICE int whh_row(int p) {
  const int w = p >> 8, n = p & 255, j = n >> 3, q = (n & 7) >> 1, e = n & 1;
  return (2 * (j & 1) + e) * kH + 64 * w + 4 * (j >> 1) + q;
}

// permuted position of the (i, f) pair of unit u; (g, o) is 8 further
EDL_DEVICE int perm_if(int u) { return (u >> 6) * 256 + 16 * ((u & 63) >> 2) + 2 * (u & 3); }

EDL_DEVICE float sigm(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
EDL_DEVICE float tanh_fast(float x) { return 2.f * sigm(2.f * x) - 1.f; }

EDL_DEVICE uint32_t pack2(float a, float b) {
  const __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&t);
}
EDL_DEVICE float2 unpack2(uint32_t v) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v)); }

// Shared prologue: W_hh of direction d permuted into sw, the clamped lengths of the tile into slen, zeroed tile bytes.
EDL_DEVICE int prologue(const __nv_bfloat16* __restrict__ whh, const int* __restrict__ lengths, uint8_t* sw, int* slen,
                        uint8_t* zero, int zero_bytes, int d, int b0, int B, int L) {
  const __nv_bfloat16* w = whh + (size_t)d * kG * kH;
  for (int i = threadIdx.x; i < kG * (kH / 8); i += kThreads) {
    const int p = i >> 4, kc = (i & 15) * 8;
    *reinterpret_cast<int4*>(sw + swz(p, kc, kG)) = *reinterpret_cast<const int4*>(w + (size_t)whh_row(p) * kH + kc);
  }
  for (int i = threadIdx.x; i < zero_bytes / 16; i += kThreads) reinterpret_cast<int4*>(zero)[i] = make_int4(0, 0, 0, 0);
  if (threadIdx.x < kRows) {
    const int b = b0 + threadIdx.x;
    slen[threadIdx.x] = b < B ? min(max(lengths[b], 0), L) : 0;
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  int mx = 0;
  for (int i = 0; i < kRows; ++i) mx = max(mx, slen[i]);
  return mx;
}

__global__ void __launch_bounds__(kThreads, 1)
lstm_fwd_kernel(const __nv_bfloat16* __restrict__ xproj, const __nv_bfloat16* __restrict__ whh,
                const int* __restrict__ lengths, __nv_bfloat16* __restrict__ hs, __nv_bfloat16* __restrict__ hn,
                __nv_bfloat16* __restrict__ gates, float* __restrict__ cs, int B, int L) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sw = smem;
  uint8_t* sh = smem + kWBytes;
  int* slen = reinterpret_cast<int*>(sh + 2 * kHTile);
  const int d = blockIdx.x, b0 = blockIdx.y * kRows;
  const int tid = threadIdx.x, wg = tid >> 7, q = tid & 3;
  const int r0 = ((tid >> 5) & 3) * 16 + ((tid & 31) >> 2);
  const int maxlen = prologue(whh, lengths, sw, slen, sh, 2 * kHTile, d, b0, B, L);
  const int len[2] = {slen[r0], slen[r0 + 8]};
  const int bb[2] = {b0 + r0, b0 + r0 + 8};
  const int ubase = 64 * wg + q;                              // unit of m is ubase + 4m
#pragma unroll
  for (int rr = 0; rr < 2; ++rr)
    if (bb[rr] < B && len[rr] == 0)
      for (int m = 0; m < 16; ++m) hn[((size_t)d * B + bb[rr]) * kH + ubase + 4 * m] = __float2bfloat16_rn(0.f);

  float acc[128];
  float c[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) c[i] = 0.f;
  const int xcol = d * kG + wg * 256 + q * 64;
  auto load_x = [&](int s) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const bool active = s < len[rr];
      const int t = d == 0 ? s : len[rr] - 1 - s;
      const int4* src = reinterpret_cast<const int4*>(xproj + ((size_t)(active ? t : 0) * B + bb[rr]) * (2 * kG) + xcol);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        int4 v = make_int4(0, 0, 0, 0);
        if (active) v = src[k];
        const uint32_t w4[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack2(w4[i]);
          acc[4 * (4 * k + i) + 2 * rr] = f.x;
          acc[4 * (4 * k + i) + 2 * rr + 1] = f.y;
        }
      }
    }
  };
  load_x(0);
  const uint32_t w_base = ptx::smem_u32(sw) + wg * 256 * 128;
  for (int s = 0; s < maxlen; ++s) {
    const uint32_t a_base = ptx::smem_u32(sh + (s & 1) * kHTile);
    ptx::wgmma_fence();
#pragma unroll
    for (int slab = 0; slab < 2; ++slab)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        ptx::WgmmaBf16<256, 0, 0>::mma(acc, ptx::make_smem_desc(a_base + slab * (kRows * 128), 16, 1024) + 2 * kk,
                                       ptx::make_smem_desc(w_base + slab * (kG * 128), 16, 1024) + 2 * kk, 1u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    uint8_t* hnext = sh + ((s + 1) & 1) * kHTile;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = r0 + 8 * rr, b = bb[rr];
      const bool active = s < len[rr];
      const int t = d == 0 ? s : len[rr] - 1 - s;
      const size_t grow = (size_t)(active ? t : s) * B + b;
      const bool last = s == len[rr] - 1;
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const int u = ubase + 4 * m;
        const float ig = sigm(acc[8 * m + 2 * rr]), fg = sigm(acc[8 * m + 2 * rr + 1]);
        const float gg = tanh_fast(acc[8 * m + 4 + 2 * rr]), og = sigm(acc[8 * m + 5 + 2 * rr]);
        const float cn = fg * c[2 * m + rr] + ig * gg;
        const float h = og * tanh_fast(cn);
        const __nv_bfloat16 hb = __float2bfloat16_rn(active ? h : 0.f);
        if (active) {
          c[2 * m + rr] = cn;
          const size_t gi = (grow * 2 + d) * kH + u;
          *reinterpret_cast<uint2*>(gates + gi * 4) = make_uint2(pack2(ig, fg), pack2(gg, og));
          cs[gi] = cn;
          if (last) hn[((size_t)d * B + b) * kH + u] = hb;
        }
        if (b < B) hs[(grow + B) * (2 * kH) + d * kH + u] = hb;
        *reinterpret_cast<__nv_bfloat16*>(hnext + swz(r, u, kRows)) = hb;
      }
    }
    if (s + 1 < maxlen) load_x(s + 1);
    ptx::fence_proxy_async_smem();
    asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory");
  }
  // zero blocks 0 and L + 1 of hs and the steps the tile never reached, for this tile's rows and direction
  const int rows_t = min(kRows, B - b0), tail = L - maxlen + 2;
  for (int i = tid; i < tail * rows_t * (kH / 8); i += kThreads) {
    const int k = i % (kH / 8), rb = (i / (kH / 8)) % rows_t, ti = i / ((kH / 8) * rows_t);
    const int blk = ti == 0 ? 0 : maxlen + ti;                // 0, then maxlen + 1 .. L + 1
    *reinterpret_cast<int4*>(hs + ((size_t)blk * B + b0 + rb) * (2 * kH) + d * kH + k * 8) = make_int4(0, 0, 0, 0);
  }
}

__global__ void __launch_bounds__(kThreads, 1)
lstm_bwd_kernel(const __nv_bfloat16* __restrict__ whh, const int* __restrict__ lengths,
                const __nv_bfloat16* __restrict__ gates, const float* __restrict__ cs,
                const __nv_bfloat16* __restrict__ dy, int64_t dy_sb, int64_t dy_st,
                const __nv_bfloat16* __restrict__ dhn, __nv_bfloat16* __restrict__ dgates, int B, int L) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sw = smem;
  uint8_t* sa = smem + kWBytes;
  int* slen = reinterpret_cast<int*>(sa + kDgTile);
  const int d = blockIdx.x, b0 = blockIdx.y * kRows;
  const int tid = threadIdx.x, wg = tid >> 7, q = tid & 3;
  const int r0 = ((tid >> 5) & 3) * 16 + ((tid & 31) >> 2);
  const int maxlen = prologue(whh, lengths, sw, slen, sa, kDgTile, d, b0, B, L);
  const int len[2] = {slen[r0], slen[r0 + 8]};
  const int bb[2] = {b0 + r0, b0 + r0 + 8};
  float acc[32], dcc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dcc[i] = 0.f;
  const uint32_t a_base = ptx::smem_u32(sa), w_base = ptx::smem_u32(sw) + wg * (kG * 128);
  for (int s = maxlen - 1; s >= 0; --s) {
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kG / 16; ++kk)
      ptx::WgmmaBf16<64, 0, 1>::mma(acc, ptx::make_smem_desc(a_base + (kk >> 2) * (kRows * 128), 16, 1024) + 2 * (kk & 3),
                                    ptx::make_smem_desc(w_base + kk * 16 * 128, kG * 128, 1024), kk != 0 ? 1u : 0u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory");   // every read of the A tile has retired
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = r0 + 8 * rr, b = bb[rr];
      const bool active = s < len[rr];
      const int t = d == 0 ? s : len[rr] - 1 - s;
      const size_t grow = (size_t)(active ? t : s) * B + b;
      const size_t gprev = (size_t)(d == 0 ? t - 1 : t + 1) * B + b;
      const bool last = s == len[rr] - 1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int u = 64 * wg + 8 * j + 2 * q;                 // units u, u + 1
        float dg[2][4];
        if (active) {
          const int4 gv = *reinterpret_cast<const int4*>(gates + ((grow * 2 + d) * kH + u) * 4);
          const float2 cc = *reinterpret_cast<const float2*>(cs + (grow * 2 + d) * kH + u);
          const float2 cp = s > 0 ? *reinterpret_cast<const float2*>(cs + (gprev * 2 + d) * kH + u) : make_float2(0.f, 0.f);
          float2 ext = make_float2(0.f, 0.f);
          if (dy != nullptr) ext = unpack2(*reinterpret_cast<const uint32_t*>(dy + b * dy_sb + (int64_t)t * dy_st + d * kH + u));
          if (last && dhn != nullptr) {
            const float2 e2 = unpack2(*reinterpret_cast<const uint32_t*>(dhn + ((size_t)d * B + b) * kH + u));
            ext.x += e2.x;
            ext.y += e2.y;
          }
          const uint32_t gw[4] = {(uint32_t)gv.x, (uint32_t)gv.y, (uint32_t)gv.z, (uint32_t)gv.w};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float2 g01 = unpack2(gw[2 * e]), g23 = unpack2(gw[2 * e + 1]);
            const float ig = g01.x, fg = g01.y, gg = g23.x, og = g23.y;
            const float c_t = e ? cc.y : cc.x, c_p = e ? cp.y : cp.x;
            const float dh = acc[4 * j + 2 * rr + e] + (e ? ext.y : ext.x);
            const float tc = tanh_fast(c_t);
            const float dc = dh * og * (1.f - tc * tc) + dcc[4 * j + 2 * rr + e];
            dg[e][0] = dc * gg * (ig * (1.f - ig));
            dg[e][1] = dc * c_p * (fg * (1.f - fg));
            dg[e][2] = dc * ig * (1.f - gg * gg);
            dg[e][3] = dh * tc * (og * (1.f - og));
            dcc[4 * j + 2 * rr + e] = dc * fg;
          }
        } else {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
#pragma unroll
            for (int g = 0; g < 4; ++g) dg[e][g] = 0.f;
            dcc[4 * j + 2 * rr + e] = 0.f;
          }
        }
        if (b < B) {
#pragma unroll
          for (int g = 0; g < 4; ++g)
            *reinterpret_cast<uint32_t*>(dgates + grow * (2 * kG) + d * kG + g * kH + u) = pack2(dg[0][g], dg[1][g]);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int p = perm_if(u + e);
          *reinterpret_cast<uint32_t*>(sa + swz(r, p, kRows)) = pack2(dg[e][0], dg[e][1]);
          *reinterpret_cast<uint32_t*>(sa + swz(r, p + 8, kRows)) = pack2(dg[e][2], dg[e][3]);
        }
      }
    }
    ptx::fence_proxy_async_smem();
    asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory");
  }
  const int rows_t = min(kRows, B - b0), tail = L - maxlen;
  for (int i = tid; i < tail * rows_t * (kG / 8); i += kThreads) {
    const int k = i % (kG / 8), rb = (i / (kG / 8)) % rows_t, t = maxlen + i / ((kG / 8) * rows_t);
    *reinterpret_cast<int4*>(dgates + ((size_t)t * B + b0 + rb) * (2 * kG) + d * kG + k * 8) = make_int4(0, 0, 0, 0);
  }
}

template <typename K>
const char* set_smem(K kernel, int bytes, bool& done) {
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return cudaGetErrorString(e);
    done = true;
  }
  return nullptr;
}

}  // namespace

bool lstm_supported(int B, int L, int E, int H) {
  return H == kLstmHidden && B >= 1 && L >= 1 && E >= 8 && E % 8 == 0 && (B + kRows - 1) / kRows <= 65535 &&
         (int64_t)(L + 2) * B < (int64_t{1} << 31) / (2 * kG);
}

const char* lstm_fwd(const void* xproj, const void* whh, const int* lengths, void* hs, void* hn, void* gates, float* cs,
                     int B, int L, cudaStream_t stream) {
  static bool attr = false;
  if (const char* e = set_smem(lstm_fwd_kernel, kFwdSmem, attr)) return e;
  lstm_fwd_kernel<<<dim3(2, (B + kRows - 1) / kRows), kThreads, kFwdSmem, stream>>>(
      static_cast<const __nv_bfloat16*>(xproj), static_cast<const __nv_bfloat16*>(whh), lengths,
      static_cast<__nv_bfloat16*>(hs), static_cast<__nv_bfloat16*>(hn), static_cast<__nv_bfloat16*>(gates), cs, B, L);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* lstm_bwd(const void* whh, const int* lengths, const void* gates, const float* cs, const void* dy,
                     int64_t dy_sb, int64_t dy_st, const void* dhn, void* dgates, int B, int L, cudaStream_t stream) {
  static bool attr = false;
  if (const char* e = set_smem(lstm_bwd_kernel, kBwdSmem, attr)) return e;
  lstm_bwd_kernel<<<dim3(2, (B + kRows - 1) / kRows), kThreads, kBwdSmem, stream>>>(
      static_cast<const __nv_bfloat16*>(whh), lengths, static_cast<const __nv_bfloat16*>(gates), cs,
      static_cast<const __nv_bfloat16*>(dy), dy_sb, dy_st, static_cast<const __nv_bfloat16*>(dhn),
      static_cast<__nv_bfloat16*>(dgates), B, L);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace edl
