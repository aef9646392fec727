// bulk.cuh -- mbarrier + 1-D bulk-copy (TMA, cp.async.bulk) wrappers shared by
// the kernels that stage contiguous global slabs in shared memory.
#pragma once
#include <stdint.h>

namespace fbbev {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t tx) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar),
               "r"(tx)
               : "memory");
}
// Spins until the phase of `bar` with `parity` has completed.  A kernel that
// issues wgmma instantiates it with DRAIN_WGMMA: the trap path then waits for
// the warpgroup's MMAs itself (ptxas would inject that wait, C7517).
template <bool DRAIN_WGMMA = false>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spins = 0; !done; ++spins) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (spins > (1u << 26)) {  // a protocol bug must not hang the GPU
      if (DRAIN_WGMMA) asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(0) : "memory");
      __trap();
    }
  }
}
// non-blocking probe of a phase
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// global -> shared 1-D bulk copy (TMA): `bytes` a multiple of 16, both
// addresses 16-byte aligned; completion is signalled on `bar` as tx bytes
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src,
                                         uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// 64-bit load from a shared-memory copy (SMEM, LDS.64) or from the global
// original (LDG.64) of the same data
template <bool SMEM>
__device__ __forceinline__ float2 ld2(const float* p) {
  if (SMEM) {
    float2 v;
    asm("ld.shared.v2.f32 {%0, %1}, [%2];"
        : "=f"(v.x), "=f"(v.y)
        : "r"(smem_u32(p)));
    return v;
  }
  return __ldg(reinterpret_cast<const float2*>(p));
}

}  // namespace fbbev
