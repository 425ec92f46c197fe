// irbpp_tma.cuh -- 1-D bulk asynchronous copies (the TMA engine's cp.async.bulk) global -> shared memory with
// an mbarrier as completion object, for sm_90a.  One elected thread arms the barrier with the byte count and
// issues the copies; the data is moved by the copy engine, not through registers; consumers wait on the
// barrier's phase parity.  Sizes and both addresses must be multiples of 16 bytes.
// Under the test-only host emulation (tests/host_harness/cuda_emu.h defines IRBPP_HOST_EMULATION) the copy is a
// memcpy by the issuing thread and the wait is a no-op: callers place a block barrier between issue and use.
#pragma once
#include <stdint.h>

namespace irbpp {

#ifdef IRBPP_HOST_EMULATION
typedef uint64_t mbarrier_t;
static inline void mbar_init(mbarrier_t*, int) {}
static inline void mbar_expect_tx(mbarrier_t*, uint32_t) {}
static inline void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, mbarrier_t*) { memcpy(dst_smem, src_gmem, bytes); }
static inline void mbar_wait(mbarrier_t*, uint32_t) {}
#else
typedef unsigned long long mbarrier_t;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(mbarrier_t* bar, int arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(arrivals));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");      // visible to the async proxy
}

// the single producer's arrival, announcing `bytes` of asynchronous transactions on this phase
__device__ __forceinline__ void mbar_expect_tx(mbarrier_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, mbarrier_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}

__device__ __forceinline__ void mbar_wait(mbarrier_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "IRBPP_MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra IRBPP_MBAR_DONE;\n"
        "bra IRBPP_MBAR_WAIT;\n"
        "IRBPP_MBAR_DONE:\n"
        "}\n" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
#endif

}  // namespace irbpp
