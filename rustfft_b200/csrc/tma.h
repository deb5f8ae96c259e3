// Thin PTX wrappers for the asynchronous-copy machinery of sm_90: mbarrier, 1-D bulk copies
// (cp.async.bulk, SASS UBLKCP) and the proxy fence between generic and async accesses of shared
// memory.  Device only; the CPU replay harness substitutes a synchronous memcpy (tests/emu).
#pragma once
#include <cstdint>

#include "common.h"

#if defined(__CUDACC__)
namespace b2 {
namespace tma {

B2_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

B2_D void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make the barrier initialisation visible to the async proxy
B2_D void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// order earlier generic-proxy accesses of shared memory before later async-proxy (TMA) accesses
B2_D void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

B2_D void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
B2_D void mbar_wait(uint64_t* bar, uint32_t parity) {
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
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completes on `bar`
B2_D void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global bulk store + its completion tracking
B2_D void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
// tiled tensor copies through a CUtensorMap (cuTensorMapEncodeTiled on the host): global -> shared completes on
// `bar`, shared -> global joins the thread's bulk group.  Coordinates are element indices, innermost first.
B2_D void tensor_g2s_3d(void* smem_dst, const void* tmap, int x, int y, int z, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
                 : "memory");
}
B2_D void tensor_g2s_4d(void* smem_dst, const void* tmap, int x, int y, int z, int w, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z), "r"(w)
                 : "memory");
}
B2_D void tensor_g2s_4d_hint(void* smem_dst, const void* tmap, int x, int y, int z, int w, uint64_t* bar, unsigned long long pol) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z), "r"(w), "l"(pol)
        : "memory");
}
B2_D void tensor_s2g_3d(const void* tmap, int x, int y, int z, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmap),
                 "r"(smem_u32(smem_src)), "r"(x), "r"(y), "r"(z)
                 : "memory");
}
// the same copies with an L2 eviction-priority hint (createpolicy, common.h: l2_evict_first / l2_evict_last)
B2_D void tensor_g2s_3d_hint(void* smem_dst, const void* tmap, int x, int y, int z, uint64_t* bar, unsigned long long pol) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z), "l"(pol)
        : "memory");
}
B2_D void tensor_s2g_3d_hint(const void* tmap, int x, int y, int z, const void* smem_src, unsigned long long pol) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4}], [%1], %5;" ::"l"(tmap),
                 "r"(smem_u32(smem_src)), "r"(x), "r"(y), "r"(z), "l"(pol)
                 : "memory");
}
B2_D void bulk_g2s_hint(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, unsigned long long pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
                 : "memory");
}
// ask L2 to fetch a contiguous global range (no destination: a pure prefetch, SASS UBLKPF); bytes a multiple of 16
B2_D void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
// plain arrival (release at CTA scope): publishes this thread's earlier shared-memory writes to the waiters
B2_D void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// non-blocking probe of a phase
B2_D bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// full generic <-> async proxy fence (all state spaces): orders a generic-proxy acquire of a flag before the
// async-proxy (TMA) reads that depend on it, and TMA-written global data before a generic-proxy release
B2_D void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// all bulk groups of this thread except the newest N have completed (writes performed, not just sources read)
template <int N> B2_D void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
template <int N> B2_D void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// named barrier among `count` threads of the CTA (consumer groups of the warp-specialised kernels)
B2_D void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
B2_D void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
B2_D void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// per-thread register budget of the calling warpgroup (every thread of all four warps executes the same one); REGS a
// multiple of 8 in [24, 256].  `dec` returns registers to the CTA's pool, `inc` blocks until the pool can supply them.
template <int REGS> B2_D void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS> B2_D void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }

}  // namespace tma
}  // namespace b2
#endif
