// fg_tma.cuh — mbarrier + 1-D TMA bulk copy (cp.async.bulk, SASS UBLKCP / SYNCS) used to stage a CTA's byte span
// into shared memory with zero per-thread load instructions, and the tile round every kernel builds on them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fg_common.cuh"

namespace fg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// global -> shared bulk copy through the TMA unit (1-D, 16-byte granules)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// The barrier of a CTA's tile and the parity its next fill completes.  One sequence for every kernel, whether it fills
// the tile once or round after round.
struct TileStage {
    uint64_t* mbar;  // 8 bytes of shared memory
    uint32_t parity;

    // thread 0 initialises the barrier; a CTA barrier must follow before load()
    __device__ __forceinline__ void init() {
        parity = 0u;
        if (threadIdx.x == 0) mbar_init(mbar, 1);
    }
    // every thread of the CTA calls it (CTA-uniform arguments); returns when the nbytes (a multiple of 16) are in the tile
    __device__ __forceinline__ void load(void* tile, const void* src, uint32_t nbytes) {
        if (threadIdx.x == 0) {
            fence_proxy_async();  // generic-proxy accesses of the previous round happen-before this async write
            mbar_expect_tx(mbar, nbytes);
            bulk_g2s(tile, src, nbytes, mbar);
        }
        mbar_wait(mbar, parity);
        parity ^= 1u;
    }
};

// The lines of one round: of the pending lines [cur, last) of a CTA, thread t looks at line cur + t.
struct TileRound {
    int o0, o1;  // this thread's line (both 0 when the thread holds none; clamped to offsets[last] past the last line)
    int base;    // span_base of line `cur`: tile byte k is input byte base + k
    int r;       // the first r pending lines fit the tile; 0: line `cur` alone does not, and what then is the kernel's own
};
// `holds_line`: this thread may hold a line this round.  Every thread of the CTA calls it: it contains a __syncthreads_count.
__device__ __forceinline__ TileRound plan_round(const int32_t* __restrict__ offsets, int cur, int last, int tile_bytes, bool holds_line) {
    const int i = cur + (int)threadIdx.x;
    TileRound t;
    t.o0 = t.o1 = 0;
    if (holds_line) {
        t.o0 = __ldg(offsets + min(i, last));
        t.o1 = __ldg(offsets + min(i + 1, last));
    }
    t.base = span_base(__ldg(offsets + cur));
    const bool fits = holds_line && i < last && t.o1 - t.base <= tile_bytes;
    t.r = __syncthreads_count(fits);  // offsets are monotone: `fits` is a prefix property
    return t;
}

}  // namespace fg
