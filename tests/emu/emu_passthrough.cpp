// emu_passthrough.cpp — the passthrough encoder's warp copy (fg_warp_copy.cuh) compiled with g++ (TEST INFRASTRUCTURE,
// see cuda_shim.h).  The 32 lanes of the warp run one after another: each stores its own bytes, so the order does not
// matter.
#define FG_HOST_EMU 1
#include <cstdint>

#include "../../flowgger_b200/csrc/fg_warp_copy.cuh"

extern "C" {

// one warp's copy of src[0, n) to dst
void emu_warp_copy(uint8_t* dst, const uint8_t* src, unsigned long long n) {
    for (int lane = 0; lane < 32; ++lane) fg::warp_copy(dst, src, n, lane);
}

// one passthrough record as the write pass stores it: the header, then the body right after it
void emu_copy_record(uint8_t* dst, const uint8_t* hdr, unsigned long long hn, const uint8_t* body, unsigned long long bn) {
    emu_warp_copy(dst, hdr, hn);
    emu_warp_copy(dst + hn, body, bn);
}

}  // extern "C"
