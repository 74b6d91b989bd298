// The tile stream of the RANSAC score kernels (motion_kernels.cu, egomotion_kernels.cu): cp.async.bulk copies of a
// pair's correspondences into shared memory, each completing on an mbarrier.
#pragma once
#include <cuda_runtime.h>

namespace ofdis {
namespace tiles {

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned a, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned a, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(a), "r"(parity)
      : "memory");
}
// one bulk copy of `bytes` (a multiple of 16) into shared memory, completing on mbarrier `mbar`
__device__ __forceinline__ void bulk_tile(unsigned dst, const void* src, unsigned bytes, unsigned mbar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(mbar)
               : "memory");
}

}  // namespace tiles
}  // namespace ofdis
