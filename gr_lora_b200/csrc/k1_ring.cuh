// k1_ring.cuh -- TMA bulk copy + mbarrier primitives (sm_90+ PTX, UBLKCP / SYNCS in SASS) and the symbol ring of the
// persistent K1 kernels (k1_warp.cuh, k1_group.cuh, k1_sf10.cuh).
#pragma once
#include "k1_fft.cuh"

namespace lb {

#ifdef __CUDACC__
LB_D uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
LB_D void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
LB_D void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LB_D void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
LB_D void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
LB_D void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
LB_D void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// A ring of NSLOT shared-memory slots of SLOT elements of T, each filled with one whole symbol (BYTES / 8 samples) by a TMA
// bulk copy.  One owner -- a warp, a group of warps or a CTA -- reads it: its symbols are first, first + stride,
// ... < n, and its it-th symbol lands in slot it % NSLOT.  init(), fill() and refill() are called by one thread of the
// owner; wait() by all of them.
template <typename T, int SLOT, int NSLOT>
struct SymbolRing {
    static constexpr uint32_t BYTES = sizeof(T) * SLOT;
    T (*slots)[SLOT];
    uint64_t *bars;                  // NSLOT mbarriers, one per slot
    const float2 *x;                 // symbol s starts at x + s * BYTES / 8
    size_t first, stride, n;

    // before the CTA barrier that precedes fill() and every wait()
    LB_D void init() const {
#pragma unroll
        for (int s = 0; s < NSLOT; s++) mbar_init(&bars[s], 1);
        fence_mbar_init();
    }
    LB_D void issue(int s, size_t sym) const {
        mbar_expect_tx(&bars[s], BYTES);
        bulk_g2s(slots[s], x + sym * (BYTES / sizeof(float2)), BYTES, &bars[s]);
    }
    // prologue: the owner's first NSLOT symbols
    LB_D void fill() const {
#pragma unroll
        for (int s = 0; s < NSLOT; s++) {
            const size_t sym = first + (size_t)s * stride;
            if (sym < n) issue(s, sym);
        }
    }
    // the slot of the owner's it-th symbol, once its bytes have landed
    LB_D T *wait(uint32_t it) const {
        const int s = it % NSLOT;
        mbar_wait(&bars[s], (it / NSLOT) & 1u);
        return slots[s];
    }
    // Every thread of the owner is done with the slot of its it-th symbol, sym: load the symbol NSLOT strides further into
    // it.  The slot was read and written through the generic proxy; the fence orders those accesses before the TMA write.
    LB_D void refill(uint32_t it, size_t sym) const {
        const size_t nxt = sym + (size_t)NSLOT * stride;
        if (nxt < n) {
            fence_proxy_async();
            issue(it % NSLOT, nxt);
        }
    }
};
#endif  // __CUDACC__

}  // namespace lb
