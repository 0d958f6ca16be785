// fg_warp_copy.cuh — one warp copies one byte span (the passthrough encoder's write pass, fg_passthrough_encode.cu).
//
// All 32 lanes store consecutive bytes of the same span: the bytes in front of the first 16-byte aligned destination
// address one per lane, then 16-byte stores (512 bytes per warp step), then the tail one byte per lane.  The source may
// sit at any alignment relative to the destination: a 16-byte store takes its bytes from the aligned 32-bit words that
// hold them, joined with a funnel shift (funnel_r), so no load reaches a word that holds no byte of the span.  Host and device code
// (the emulation tests compile this header with g++ and run the lanes one after another).
#pragma once
#include <stdint.h>
#ifdef FG_HOST_EMU
#include "../../tests/emu/cuda_shim.h"
#endif

namespace fg {

// the low 32 bits of hi:lo >> sh (0 < sh < 32): one funnel shift (SHF) on the device, the same expression on the host
__host__ __device__ __forceinline__ uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {
    return (uint32_t)((((unsigned long long)hi << 32) | lo) >> sh);
}

// lane `lane` of a warp's copy of src[0, n) to dst[0, n); every lane of the warp calls it with the same arguments
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, unsigned long long n, int lane) {
    const unsigned long long mis = (unsigned long long)(16u - ((uint32_t)(uintptr_t)dst & 15u)) & 15ull;
    const unsigned long long head = mis < n ? mis : n;
    if ((unsigned long long)lane < head) dst[lane] = src[lane];
    uint8_t* d = dst + head;
    const uint8_t* s = src + head;
    const unsigned long long body = (n - head) & ~15ull;
    const uint32_t sa = (uint32_t)(uintptr_t)s & 15u, sh = (sa & 3u) * 8u;
    const unsigned long long k0 = 16ull * (unsigned)lane;
    if (sa == 0u) {
        for (unsigned long long k = k0; k < body; k += 512ull)
            *reinterpret_cast<uint4*>(d + k) = *reinterpret_cast<const uint4*>(s + k);
    } else if (sh == 0u) {  // 4-byte aligned source
        for (unsigned long long k = k0; k < body; k += 512ull) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(s + k);
            *reinterpret_cast<uint4*>(d + k) = uint4{w[0], w[1], w[2], w[3]};
        }
    } else {  // the five words that hold s[k, k + 16): the first and last hold bytes of this chunk, no more
        for (unsigned long long k = k0; k < body; k += 512ull) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(s + k - (sh >> 3));
            const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
            *reinterpret_cast<uint4*>(d + k) =
                uint4{funnel_r(w0, w1, sh), funnel_r(w1, w2, sh), funnel_r(w2, w3, sh), funnel_r(w3, w4, sh)};
        }
    }
    const unsigned long long tail = n - head - body;  // < 16
    if ((unsigned long long)lane < tail) d[body + lane] = s[body + lane];
}

}  // namespace fg
