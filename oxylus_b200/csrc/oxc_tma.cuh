// oxc_tma.cuh — the Hopper bulk asynchronous copy engine (TMA) in its 1-D form: cp.async.bulk global -> shared with
// completion on an mbarrier (SASS: UBLKCP + SYNCS), plus an L1 prefetch hint.  Used by the raster (micro-index runs) and
// available to the cull kernels.
#pragma once
#include "oxc_exact.cuh"

namespace oxc {

// ---- TMA (bulk async copy engine): 1-D cp.async.bulk global -> shared, completion on an mbarrier ----
OXC_DI uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
OXC_DI void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
OXC_DI void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
OXC_DI void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
OXC_DI void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
OXC_DI void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

#ifdef OXC_HOST_SOUNDNESS_HARNESS
OXC_DI void prefetch_l1(const void*) {} // host builds of the headers (tests/): a hint has no result
#else
OXC_DI void prefetch_l1(const void* ptr) { asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr)); }
#endif

} // namespace oxc
