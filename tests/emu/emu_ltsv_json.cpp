// emu_ltsv_json.cpp — CPU emulation of the fused LTSV encoder's GELF string path (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's json_unescape_step (fg_gelf.cuh, the decoder's KeyIter unescape) and ltsv_escape4
// (fg_ltsv_text.cuh, LTSVString::insert's replacements) with g++ and drives them over one JSON string body the way
// run_ltsv (fg_ltsv_encode.cu) does for a segment of kind SK_JSON_VAL / SK_JSON_KEY: a word of four source bytes when
// four remain and none is a backslash, else one unescape step (1..4 output bytes), and the word then through
// ltsv_escape4.  The loop restates run_ltsv's, as emu_json.cpp restates gelf_write_kernel's.
#define FG_HOST_EMU 1
#include <cstdint>

#include "cuda_shim.h"
#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_gelf.cuh"
#include "../../flowgger_b200/csrc/fg_ltsv_text.cuh"

extern "C" {

// body p[0, len) (a validated JSON string body; mode2: the line went through the newline retry) -> the LTSV text of its
// unescaped bytes as a key (key != 0) or a value, in out[0, ret); -1 when out is too small
int emu_ltsv_json(const uint8_t* p, int len, int mode2, int key, uint8_t* out, int cap) {
    int k = 0, n = 0;
    while (k < len) {
        uint32_t w = p[k];
        int c = 1;
        if (k + 4 <= len) {
            w |= ((uint32_t)p[k + 1] << 8) | ((uint32_t)p[k + 2] << 16) | ((uint32_t)p[k + 3] << 24);
            c = 4;
        }
        if (c == 1 || fg::ltsv_eq4(w, 0x5C5C5C5Cu)) c = fg::json_unescape_step(p, k, len, mode2 != 0, w);
        else k += c;
        w = fg::ltsv_escape4(w, key != 0);
        if (n + c > cap) return -1;
        for (int j = 0; j < c; ++j) out[n++] = (uint8_t)(w >> (8 * j));
    }
    return n;
}

}  // extern "C"
