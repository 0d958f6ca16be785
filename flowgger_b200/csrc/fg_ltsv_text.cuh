// fg_ltsv_text.cuh — the byte replacements of LTSVString::insert (ltsv_encoder.rs:43-59): in a key '\n' and '\t' become
// ' ' and ':' becomes '_'; in a value '\t' and '\n' become ' '.  Nothing else changes and every byte stays one byte, so
// a span's length is its text's length.
#pragma once
#include <stdint.h>

#include "fg_simt.cuh"

namespace fg {

// 0x80 in every byte of w equal to b (b replicated in all four bytes)
FG_DEV uint32_t ltsv_eq4(uint32_t w, uint32_t b4) {
    const uint32_t x = w ^ b4;
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}
// 0x80 in every byte of w the LTSV text replaces (key: also ':')
FG_DEV uint32_t ltsv_flags4(uint32_t w, bool key) {
    uint32_t f = ltsv_eq4(w, 0x09090909u) | ltsv_eq4(w, 0x0A0A0A0Au);
    if (key) f |= ltsv_eq4(w, 0x3A3A3A3Au);
    return f;
}
// the four bytes of w with the replacements made
FG_DEV uint32_t ltsv_escape4(uint32_t w, bool key) {
    const uint32_t ws = (ltsv_eq4(w, 0x09090909u) | ltsv_eq4(w, 0x0A0A0A0Au)) >> 7;  // 0x01 per byte to become ' '
    w = (w & ~(ws * 0xFFu)) | (ws * 0x20u);
    if (key) {
        const uint32_t wc = ltsv_eq4(w, 0x3A3A3A3Au) >> 7;
        w = (w & ~(wc * 0xFFu)) | (wc * 0x5Fu);
    }
    return w;
}

}  // namespace fg
