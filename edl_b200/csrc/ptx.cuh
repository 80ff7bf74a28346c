// Thin inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the GEMM / conv
// kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma (wgmma.cuh) and its shared-memory matrix
// descriptor.  Bit layouts follow the PTX ISA chapter "Asynchronous warpgroup level matrix instructions".
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace edl {
namespace ptx {

EDL_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
EDL_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
EDL_DEVICE void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
EDL_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
EDL_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
EDL_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking poll (try_wait may suspend the thread for a system-dependent time)
EDL_DEVICE bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
EDL_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// shared-memory accesses by 32-bit shared address (no generic-pointer 64-bit address arithmetic)
EDL_DEVICE uint32_t lds32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
EDL_DEVICE void sts128(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// One lane of the (fully active) warp; the same lane every time for the same mask.
EDL_DEVICE bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- TMA
EDL_DEVICE void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
EDL_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
EDL_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
EDL_DEVICE void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
      : "memory");
}
EDL_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
EDL_DEVICE void tma_store_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
EDL_DEVICE void tma_store_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// make generic-proxy smem writes visible to the async proxy (TMA store source)
EDL_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor, SWIZZLE_128B.  (addr, LBO, SBO are byte values.)
//   K-major : rows of 128 B (64 bf16), 8-row groups 1024 B apart -> SBO = 1024, LBO unused (1)
//   MN-major: [k rows][64 mn elems = 128 B]; 8-k-row groups 1024 B apart -> SBO = 1024,
//             64-element MN chunks LBO bytes apart
// kSwizzleBytes = 64: SWIZZLE_64B (layout type 2), the same with rows of 64 B (32 bf16) and 8-row groups 512 B apart
// (SBO = 512); the matching tensor map is CU_TENSOR_MAP_SWIZZLE_64B.
template <int kSwizzleBytes = 128>
EDL_DEVICE uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  static_assert(kSwizzleBytes == 128 || kSwizzleBytes == 64, "128B or 64B swizzle");
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(kSwizzleBytes == 128 ? 1 : 2) << 62;
  return d;
}

// Same, with an explicit "matrix base offset" (bits 49..51): the PTX ISA asks for ((start address >> 7) & 7) when the
// matrix does not start on the 1024-byte boundary of the 128B-swizzle repeating pattern.
EDL_DEVICE uint64_t make_smem_desc_bo(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t base_offset) {
  return make_smem_desc(saddr, lbo_bytes, sbo_bytes) | ((uint64_t)(base_offset & 7u) << 49);
}

}  // namespace ptx
}  // namespace edl
