// sm_90 mbarrier and bulk-copy (TMA engine) wrappers around inline PTX, shared by the persistent Schur kernels
// (ba_schur_pipe.cuh) and the tensor-core matcher (match_tc.cu).  Each caller keeps its own arrival protocol.
#pragma once

#include <cstdint>

namespace osfm {

// A protocol bug must surface as a trapped kernel, never as a hung GPU: an mbarrier wait gives up after this many
// SM clocks (seconds at H100 clocks; a legitimate wait in these kernels lasts microseconds).
constexpr long long MBAR_TIMEOUT_CLOCKS = 8000000000LL;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive and expect `bytes` more from bulk copies that complete on this barrier
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Wait for the phase of the given parity to complete.  On a timeout, sets *err_flag (when given) and traps.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag = nullptr) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long t0 = 0;
  int spins = 0;
  // try_wait suspends the thread for a hardware-defined time slice before it reports failure, so the loop is
  // cheap; the clock is only consulted every 1024 failed slices.  (Other shapes of this loop make ba_schur_pipe,
  // which runs at its 96-register bound, spill.)
  while (true) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    if ((++spins & 1023) == 0) {
      if (t0 == 0) t0 = clock64();
      else if (clock64() - t0 > MBAR_TIMEOUT_CLOCKS) {
        if (err_flag) atomicExch(err_flag, 1);
        __trap();
      }
    }
  }
}
// global -> shared bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned), completing on `bar`
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

}  // namespace osfm
