// tma.cuh — mbarrier and bulk-copy (TMA, SASS UBLKCP) helpers of the K2 ring (k2_ring.cu).
#pragma once

#include "common.cuh"

namespace bz {

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// BZ_MBAR_HINT_NS (A/B builds): suspend-time hint of try_wait.  Without it the hardware wait is
// short and a waiting warp re-issues the probe ~28 times per tile (ncu, n = 25: SYNCS + BRA + YIELD
// = 11 % of the executed instructions, on the schedulers the working warps need).
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
#ifdef BZ_MBAR_HINT_NS
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity), "r"((unsigned)BZ_MBAR_HINT_NS) : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#endif
}

}  // namespace bz
