// emu_ltsv_text.cpp — CPU emulation of the LTSV encoder's text routines (TEST INFRASTRUCTURE, see cuda_shim.h): Rust's
// Display for f64 (fg_ftoa.cuh) and the key / value replacements of LTSVString::insert (fg_ltsv_text.cuh), compiled
// with g++ from the product headers.
#define FG_HOST_EMU 1
#include <cstdint>

#include "cuda_shim.h"
#include "../../flowgger_b200/csrc/fg_ftoa.cuh"
#include "../../flowgger_b200/csrc/fg_ltsv_text.cuh"

extern "C" {

// the text of each v[i] one after the other in out; lens[i] its length; returns the total, -1 when out is too small
long long emu_f64_display(const double* v, long long n, uint8_t* out, long long cap, int32_t* lens) {
    long long at = 0;
    for (long long i = 0; i < n; ++i) {
        fg::FtoaText t;
        fg::f64_display(v[i], t);
        if (at + t.len() > cap) return -1;
        for (int k = 0; k < t.len(); ++k) out[at + k] = t.at(k);
        lens[i] = t.len();
        at += t.len();
    }
    return at;
}

// p[0, len) as an LTSV key (key != 0) or value, four bytes at a time as the byte loop does, the tail one by one
void emu_ltsv_escape(const uint8_t* p, int len, int key, uint8_t* out) {
    int k = 0;
    for (; k + 4 <= len; k += 4) {
        uint32_t w = 0;
        for (int j = 0; j < 4; ++j) w |= (uint32_t)p[k + j] << (8 * j);
        if (fg::ltsv_flags4(w, key != 0)) w = fg::ltsv_escape4(w, key != 0);
        for (int j = 0; j < 4; ++j) out[k + j] = (uint8_t)(w >> (8 * j));
    }
    for (; k < len; ++k) out[k] = (uint8_t)fg::ltsv_escape4(p[k], key != 0);
}

}  // extern "C"
