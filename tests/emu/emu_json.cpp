// emu_json.cpp — CPU emulation of the fused GELF encoder's string re-encoding (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's json_transcode_step (fg_gelf.cuh: the decoder's KeyIter unescape + json_escape_of) with g++ and
// drives it over a whole JSON string body the way gelf_write_kernel's byte loop does for an escaped span: four source
// bytes at a time while they hold no backslash and no byte to escape, else one step.
#define FG_HOST_EMU 1
#include <cstdint>

#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_gelf.cuh"

extern "C" {

// body p[0, len) (a validated JSON string body; mode2: the line went through the newline retry) -> serde_json text in
// out[0, ret); -1 when out is too small
int emu_json_transcode(const uint8_t* p, int len, int mode2, uint8_t* out, int cap) {
    int k = 0, n = 0;
    while (k < len) {
        if (k + 4 <= len) {
            bool plain = true;
            for (int j = 0; j < 4; ++j) plain = plain && p[k + j] != '\\' && fg::json_escape_of(p[k + j]) == 0u && p[k + j] >= 0x20u;
            if (plain) {
                if (n + 4 > cap) return -1;
                for (int j = 0; j < 4; ++j) out[n++] = p[k++];
                continue;
            }
        }
        uint32_t w;
        const int c = fg::json_transcode_step(p, k, len, mode2 != 0, w);
        if (n + c > cap) return -1;
        for (int j = 0; j < c; ++j) out[n++] = (uint8_t)(w >> (8 * j));
    }
    return n;
}

}  // extern "C"
