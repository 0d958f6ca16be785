// fg_out_frame.cuh — output.framing (merger/*.rs), applied by the fused GELF encoder to every record it writes.
//
// The reference's Output hands each encoded record to its Merger before it writes it (output/file_output.rs:209-210,
// tls_output.rs:109-110, debug_output.rs:28-29):
//   line    record "\n"                     (line_merger.rs:14)
//   nul     record "\0"                     (nul_merger.rs:14)
//   syslen  "{L + 1} " record "\n"           (syslen_merger.rs:15-28: L = the record's length, the +1 counts the "\n")
// A record the decoder rejected is never sent, so it gets no frame.  Host and device code (the emulation tests compile
// this header with g++).
#pragma once
#include <stdint.h>
#ifdef FG_HOST_EMU
#include "../../tests/emu/cuda_shim.h"
#endif

namespace fg {

enum OutFraming { kOutNone = 0, kOutLine = 1, kOutNul = 2, kOutSyslen = 3 };  // = fg_out_framing

// decimal digits of v
__host__ __device__ __forceinline__ int dec_digits(unsigned long long v) {
    int d = 1;
    for (; v >= 10ull; v /= 10ull) ++d;
    return d;
}

// syslen's prefix of a record of `len` bytes: the decimal of len + 1 and one space, written to out[0, ret) (ret <= 21)
__host__ __device__ __forceinline__ int syslen_prefix(unsigned long long len, uint8_t* out) {
    unsigned long long v = len + 1ull;
    const int d = dec_digits(v);
    for (int k = d - 1; k >= 0; --k, v /= 10ull) out[k] = (uint8_t)('0' + (uint32_t)(v % 10ull));
    out[d] = ' ';
    return d + 1;
}

// bytes written for a record of `len` bytes
__host__ __device__ __forceinline__ unsigned long long framed_len(unsigned long long len, int framing) {
    if (framing == kOutSyslen) return (unsigned long long)dec_digits(len + 1ull) + 1ull + len + 1ull;
    return len + (framing == kOutNone ? 0ull : 1ull);
}

// the record length `len` of framed_len(len, framing) == f: with m = len + 1, f - 1 = m + digits(m) rises strictly with
// m, and digits(m) is digits(f - 1) or one less
__host__ __device__ __forceinline__ unsigned long long unframed_len(unsigned long long f, int framing) {
    if (framing != kOutSyslen) return f - (framing == kOutNone ? 0ull : 1ull);
    const int d = dec_digits(f - 1ull);
    const unsigned long long m = f - 1ull - (unsigned long long)d;
    return (dec_digits(m) == d ? m : m + 1ull) - 1ull;
}

// The frame of a record whose framed bytes, `framed` of them, start at `out`: the suffix byte at the end and (syslen) the
// prefix at the start are stored; returns where the record's own bytes go
__host__ __device__ __forceinline__ uint8_t* frame_record(int framing, unsigned long long framed, uint8_t* out) {
    if (framing == kOutNone) return out;
    out[framed - 1ull] = framing == kOutNul ? (uint8_t)0 : (uint8_t)'\n';
    if (framing != kOutSyslen) return out;
    return out + syslen_prefix(unframed_len(framed, kOutSyslen), out);
}

}  // namespace fg
