// tma.cuh — bulk asynchronous copies (cp.async.bulk, the 1-D TMA path, SASS UBLKCP) + mbarrier helpers.
//
// Why: the operators here are HBM-bound streams mixed with random gathers.  One 8-byte LDG in flight per thread
// cannot cover HBM latency (a plain probe kernel stalls on long_scoreboard).  Bulk copies are issued by one elected thread, need no registers for
// the data in flight, bypass the LSU/L1 miss path, and complete on an mbarrier, so every CTA keeps several
// 16-32 KB tiles in flight regardless of occupancy.
#pragma once
#include <cstdint>

namespace tg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      "  .reg .pred p;\n"
      "  mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "  selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Every lane performs its own acquire, then the warp reconverges: try_wait may release lanes of one warp at
// different times, and the CTA-wide __syncthreads() that follows in the kernels is an ALIGNED barrier — executing it
// with a diverged warp is undefined (the barrier can release early and the stage be refilled under lanes that have
// not read it yet).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
  __syncwarp();
}

__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_normal() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// global → shared bulk copy; src/dst 16-byte aligned, bytes a multiple of 16; completion on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar,
                                         unsigned long long policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

}  // namespace tg
