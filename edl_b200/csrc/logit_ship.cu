// Teacher -> student transport over NVSwitch peer memory, fused with the distillation loss
// (SURVEY K13 + K6).
//
// Reference path being replaced: every teacher batch travels student -> Paddle Serving (brpc/TCP,
// 9.6 MB up) -> teacher GPU -> host -> TCP (64 KB down) -> three pickle hops -> host numpy -> H2D ->
// softmax_with_cross_entropy (python/edl/distill/distill_worker.py:243-308,
// example/distill/resnet/train_with_fleet.py:254-259).  When teacher and student GPUs share an
// NVSwitch domain none of that is needed:
//
//   peer_ship      : a rank pushes a payload (e.g. the student's input batch for the teacher) into a
//                    ring slot in the PEER's HBM with 128-bit stores and publishes a sequence flag.
//   logit_ship     : the teacher pushes its logits [B, C] into the student's slot AND, in the same
//                    pass, computes the per-row softmax statistics (max, log-sum-exp at temperature
//                    T) the loss needs, so the student never re-reduces the teacher distribution.
//   soft_ce_recv   : the student's loss kernel acquires the flag (bounded spin), reads the slot from
//                    local HBM and evaluates  -sum softmax(t/T) * log softmax(z/Ts)  per row, writing
//                    the loss and the row stats for the backward kernel (loss.cu soft_ce_bwd, mode 1).
//   slot_ack       : the student tells the teacher the slot may be reused (flow control).
//
// No NCCL call and no RPC on this path; sequence numbers are passed by the host (monotonic) or read
// from device memory so that both sides can be captured in CUDA graphs.
#include "comm.cuh"
#include "kernels.h"

namespace edl {
namespace {

constexpr int kShipThreads = 256;
constexpr int kRowThreads = 128;

EDL_DEVICE float blk_sum(float v, float* sh, int nwarps) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < nwarps; ++i) r += sh[i];
  return r;
}
EDL_DEVICE float blk_max(float v, float* sh, int nwarps) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = -INFINITY;
  for (int i = 0; i < nwarps; ++i) r = fmaxf(r, sh[i]);
  return r;
}

// Generic payload push: dst (peer pointer) <- src (local), then flag <- seq (release, system scope)
// once every block has finished.  `done` is a local zero-initialised counter re-armed by the last block.
__global__ void __launch_bounds__(kShipThreads)
peer_ship_kernel(const int4* __restrict__ src, int4* __restrict__ dst_peer, int64_t nvec,
                 uint32_t* __restrict__ flag_peer, const uint32_t* __restrict__ seq_ptr, uint32_t seq_imm,
                 unsigned int* __restrict__ done) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x)
    st_peer(dst_peer + i, src[i]);
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {
      *done = 0u;
      __threadfence_system();
      st_release_sys(flag_peer, seq_ptr != nullptr ? *seq_ptr : seq_imm);
    }
  }
}

// One block per row: ship the logits row to the peer slot, compute (max, lse) at temperature T.
// `vec` (decided on the host): every row of source and slot starts on a 16-byte boundary, so the
// copy moves 8 logits per 128-bit access; otherwise (C % 8 != 0, or an unaligned base) it goes
// element by element.
__global__ void __launch_bounds__(kRowThreads)
logit_ship_kernel(const __nv_bfloat16* __restrict__ logits, __nv_bfloat16* __restrict__ slot_peer,
                  float* __restrict__ stats_peer /* [B,2] */, int B, int C, int vec, float inv_temp,
                  uint32_t* __restrict__ flag_peer, const uint32_t* __restrict__ seq_ptr, uint32_t seq_imm,
                  unsigned int* __restrict__ done) {
  __shared__ float sh[kRowThreads / 32];
  const int row = blockIdx.x;
  const __nv_bfloat16* src = logits + (int64_t)row * C;
  __nv_bfloat16* dst = slot_peer + (int64_t)row * C;
  float mx = -INFINITY;
  const int nvec = vec ? C / 8 : 0;
  for (int v = threadIdx.x; v < nvec; v += kRowThreads) {
    const bf16x8 x = ld_vec(src + v * 8);
    st_peer(reinterpret_cast<int4*>(dst) + v, *reinterpret_cast<const int4*>(&x));
    float f[8];
    unpack8(x, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) mx = fmaxf(mx, f[i] * inv_temp);
  }
  for (int j = nvec * 8 + threadIdx.x; j < C; j += kRowThreads) {
    dst[j] = src[j];
    mx = fmaxf(mx, __bfloat162float(src[j]) * inv_temp);
  }
  mx = blk_max(mx, sh, kRowThreads / 32);
  float s = 0.f;
  for (int j = threadIdx.x; j < C; j += kRowThreads) s += __expf(__bfloat162float(src[j]) * inv_temp - mx);
  s = blk_sum(s, sh, kRowThreads / 32);
  if (threadIdx.x == 0) {
    stats_peer[row * 2 + 0] = mx;
    stats_peer[row * 2 + 1] = mx + __logf(s);
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {
      *done = 0u;
      __threadfence_system();
      st_release_sys(flag_peer, seq_ptr != nullptr ? *seq_ptr : seq_imm);
    }
  }
}

// Spin until *flag >= seq (wrap-safe) or the timeout elapses; returns false on timeout.
EDL_DEVICE bool wait_flag(const uint32_t* flag, uint32_t seq, unsigned long long timeout_ns, uint32_t* err) {
  const unsigned long long t0 = globaltimer_ns();
  while ((int)(ld_acquire_sys(flag) - seq) < 0) {
    if (timeout_ns != 0 && globaltimer_ns() - t0 > timeout_ns) {
      if (err != nullptr) atomicExch(err, 1u);
      return false;
    }
  }
  return true;
}

// Student side: loss over a received slot.  One block per row; thread 0 of each block acquires the flag.
// row_stats out: [B,4] = (zmax, lse_z, psum=1, lse_t) -- the layout soft_ce_bwd (mode 1) consumes.
template <typename LT>
__global__ void __launch_bounds__(kRowThreads)
soft_ce_recv_kernel(const LT* __restrict__ logits, const __nv_bfloat16* __restrict__ slot,
                    const float* __restrict__ slot_stats, const uint32_t* __restrict__ flag,
                    const uint32_t* __restrict__ seq_ptr, uint32_t seq_imm, float* __restrict__ loss_out,
                    float* __restrict__ row_stats, int B, int C, float inv_ts, float inv_tt, int kl,
                    float loss_scale, unsigned long long timeout_ns, uint32_t* __restrict__ err) {
  __shared__ float sh[kRowThreads / 32];
  __shared__ int ok;
  const int row = blockIdx.x;
  if (threadIdx.x == 0) ok = wait_flag(flag, seq_ptr != nullptr ? *seq_ptr : seq_imm, timeout_ns, err) ? 1 : 0;
  __syncthreads();
  if (!ok) return;
  const LT* z = logits + (int64_t)row * C;
  const __nv_bfloat16* t = slot + (int64_t)row * C;
  auto ldz = [&](int j) -> float {
    if constexpr (sizeof(LT) == 2) return __bfloat162float(z[j]) * inv_ts;
    else return (float)z[j] * inv_ts;
  };
  float zmax = -INFINITY;
  for (int j = threadIdx.x; j < C; j += kRowThreads) zmax = fmaxf(zmax, ldz(j));
  zmax = blk_max(zmax, sh, kRowThreads / 32);
  float zsum = 0.f;
  for (int j = threadIdx.x; j < C; j += kRowThreads) zsum += __expf(ldz(j) - zmax);
  zsum = blk_sum(zsum, sh, kRowThreads / 32);
  const float lse = zmax + __logf(zsum);
  float tlse;
  if (slot_stats != nullptr) {
    tlse = slot_stats[row * 2 + 1];
  } else {
    // the slot was filled by the fused GEMM->ship epilogue (raw logits only): reduce the teacher row here
    float tmax = -INFINITY;
    for (int j = threadIdx.x; j < C; j += kRowThreads) tmax = fmaxf(tmax, __bfloat162float(t[j]) * inv_tt);
    tmax = blk_max(tmax, sh, kRowThreads / 32);
    float tsum = 0.f;
    for (int j = threadIdx.x; j < C; j += kRowThreads) tsum += __expf(__bfloat162float(t[j]) * inv_tt - tmax);
    tsum = blk_sum(tsum, sh, kRowThreads / 32);
    tlse = tmax + __logf(tsum);
  }
  float pz = 0.f, plogp = 0.f;
  for (int j = threadIdx.x; j < C; j += kRowThreads) {
    const float lt = __bfloat162float(t[j]) * inv_tt - tlse;
    const float p = __expf(lt);
    pz = fmaf(p, ldz(j), pz);
    if (kl) plogp = fmaf(p, lt, plogp);
  }
  pz = blk_sum(pz, sh, kRowThreads / 32);
  if (kl) plogp = blk_sum(plogp, sh, kRowThreads / 32);
  if (threadIdx.x == 0) {
    atomicAdd(loss_out, (lse - pz + (kl ? plogp : 0.f)) * loss_scale / (float)B);
    row_stats[row * 4 + 0] = zmax;
    row_stats[row * 4 + 1] = lse;
    row_stats[row * 4 + 2] = 1.f;
    row_stats[row * 4 + 3] = tlse;
  }
}

__global__ void slot_ack_kernel(uint32_t* __restrict__ ack_peer, const uint32_t* __restrict__ seq_ptr,
                                uint32_t seq_imm) {
  __threadfence_system();
  st_release_sys(ack_peer, seq_ptr != nullptr ? *seq_ptr : seq_imm);
}

__global__ void wait_flag_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ seq_ptr,
                                 uint32_t seq_imm, unsigned long long timeout_ns, uint32_t* __restrict__ err) {
  wait_flag(flag, seq_ptr != nullptr ? *seq_ptr : seq_imm, timeout_ns, err);
}

}  // namespace

void peer_ship(const void* src, void* dst_peer, int64_t nbytes, void* flag_peer, const void* seq_ptr,
               uint32_t seq_imm, void* done_counter, cudaStream_t s) {
  const int64_t nvec = nbytes / 16;
  int64_t blocks = (nvec + kShipThreads - 1) / kShipThreads;
  if (blocks > 64) blocks = 64;
  if (blocks < 1) blocks = 1;
  peer_ship_kernel<<<(int)blocks, kShipThreads, 0, s>>>(
      reinterpret_cast<const int4*>(src), reinterpret_cast<int4*>(dst_peer), nvec,
      reinterpret_cast<uint32_t*>(flag_peer), reinterpret_cast<const uint32_t*>(seq_ptr), seq_imm,
      reinterpret_cast<unsigned int*>(done_counter));
}

void logit_ship(const void* logits, void* slot_peer, float* stats_peer, int B, int C, float temperature,
                void* flag_peer, const void* seq_ptr, uint32_t seq_imm, void* done_counter, cudaStream_t s) {
  const bool vec = C % 8 == 0 && reinterpret_cast<uintptr_t>(logits) % 16 == 0 &&
                   reinterpret_cast<uintptr_t>(slot_peer) % 16 == 0;
  logit_ship_kernel<<<B, kRowThreads, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(logits), reinterpret_cast<__nv_bfloat16*>(slot_peer), stats_peer, B,
      C, vec ? 1 : 0, 1.f / temperature, reinterpret_cast<uint32_t*>(flag_peer),
      reinterpret_cast<const uint32_t*>(seq_ptr), seq_imm, reinterpret_cast<unsigned int*>(done_counter));
}

void soft_ce_recv(const void* logits, bool logits_bf16, const void* slot, const float* slot_stats, const void* flag,
                  const void* seq_ptr, uint32_t seq_imm, float* loss_out, float* row_stats, int B, int C,
                  float s_temp, float t_temp, bool kl, float loss_scale, double timeout_s, void* err,
                  cudaStream_t s) {
  const unsigned long long tns = (unsigned long long)(timeout_s * 1e9);
  if (logits_bf16)
    soft_ce_recv_kernel<__nv_bfloat16><<<B, kRowThreads, 0, s>>>(
        reinterpret_cast<const __nv_bfloat16*>(logits), reinterpret_cast<const __nv_bfloat16*>(slot), slot_stats,
        reinterpret_cast<const uint32_t*>(flag), reinterpret_cast<const uint32_t*>(seq_ptr), seq_imm, loss_out,
        row_stats, B, C, 1.f / s_temp, 1.f / t_temp, kl ? 1 : 0, loss_scale, tns, reinterpret_cast<uint32_t*>(err));
  else
    soft_ce_recv_kernel<float><<<B, kRowThreads, 0, s>>>(
        reinterpret_cast<const float*>(logits), reinterpret_cast<const __nv_bfloat16*>(slot), slot_stats,
        reinterpret_cast<const uint32_t*>(flag), reinterpret_cast<const uint32_t*>(seq_ptr), seq_imm, loss_out,
        row_stats, B, C, 1.f / s_temp, 1.f / t_temp, kl ? 1 : 0, loss_scale, tns, reinterpret_cast<uint32_t*>(err));
}

void slot_ack(void* ack_peer, const void* seq_ptr, uint32_t seq_imm, cudaStream_t s) {
  slot_ack_kernel<<<1, 1, 0, s>>>(reinterpret_cast<uint32_t*>(ack_peer), reinterpret_cast<const uint32_t*>(seq_ptr),
                                  seq_imm);
}

void wait_flag_async(const void* flag, const void* seq_ptr, uint32_t seq_imm, double timeout_s, void* err,
                     cudaStream_t s) {
  wait_flag_kernel<<<1, 1, 0, s>>>(reinterpret_cast<const uint32_t*>(flag), reinterpret_cast<const uint32_t*>(seq_ptr),
                                   seq_imm, (unsigned long long)(timeout_s * 1e9), reinterpret_cast<uint32_t*>(err));
}

}  // namespace edl
