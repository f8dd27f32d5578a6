// tma.cuh -- TMA bulk copies (cp.async.bulk global -> shared, completion counted on an mbarrier) as inline PTX for sm_90a (H100).
// One thread arms the barrier with the byte count (mbar_expect_tx) and issues the copies (bulk_g2s: 16-byte granularity and
// alignment on both sides); every thread that reads the data waits on the barrier's phase (mbar_wait).  SASS: UBLKCP / SYNCS.
// Used by K1 (its automaton tables).  (Round 2 also staged a hot slice of the pair table for bpe_merge_kernel this way: slower,
// removed.)
// The CPU SIMT emulator has no asynchronous proxy: its builds copy with plain loops instead.
#pragma once
#include <stdint.h>

namespace cfbpe {
#if !defined(CUSIM_EMULATOR)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}"
                 ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
#endif

}  // namespace cfbpe
